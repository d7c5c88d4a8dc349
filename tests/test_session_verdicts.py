"""CPU tests of how the two units of a fused GG20 offline session share their proof checks (csrc/gg20_rounds.cuh, declared
shortcut 10 of DESIGN.md section 4): each Pedersen, PDL-with-slack and HomoElGamal proof is verified once, on its prover's unit,
and the peer's finish kernel reads that verdict.  The round kernels run on the host harness (tests/host_harness/
session_harness.cpp) over a hand-built arena of three sessions:

- the check kernels write only their own unit's verdict byte (14, 16, 18);
- with one verdict false on exactly one unit, the finish kernels put the status the two-check version gives (every unit checks
  both proofs of its session, first failure wins) on both units of that session and on no other unit;
- R from gg20_r4_pre is bit-identical on the two units of a session, also for a sum of the Gammas at infinity, equal Gammas,
  k = 0, alpha = 0 mod q and a delta sum of zero, which is what lets one unit's verdict stand for the peer's."""
import ctypes
import os
import random
import subprocess

import numpy as np
import pytest

import __graft_entry__ as entry
from oracle import gg20_oracle as o

HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "host_harness")
OK, INVALID_KEY, PDL, PHASE5, PHASE6, PROOF = 0, 2, 6, 7, 8, 10
KEY_SIZE = [64, 128, 64, 64, 64, 64, 64, 32, 32, 32, 32, 32, 32, 32, 32, 32, 64, 32, 32, 8, 16]
R3_CHECK, R3_FINISH, R4_PRE, R5_CHECK, R5_FINISH, R6_CHECK, R6 = range(7)
PED, PDL_BYTE, HEG = 14, 16, 18
RND_K, RND_L, RND_PDL_ALPHA, RND_HEG_S1, RND_HEG_S2 = 8, 1120, 1144, 1392, 1400


def L(v, k):
    return np.frombuffer(int(v).to_bytes(4 * k, "little"), dtype=np.uint32).copy()


def I(a):
    return int.from_bytes(np.ascontiguousarray(a).tobytes(), "little")


def pt16(p):
    return np.zeros(16, np.uint32) if p is None else np.concatenate([L(p[0], 8), L(p[1], 8)])


def from16(a):
    return None if not a.any() else (I(a[:8]), I(a[8:16]))


@pytest.fixture(scope="module")
def hs():
    so = os.path.join(HERE, "libsession_host.so")
    src = os.path.join(HERE, "session_harness.cpp")
    deps = [src] + [os.path.join(entry.CSRC, f) for f in os.listdir(entry.CSRC) if f.endswith((".cuh", ".h"))] + \
           [os.path.join(entry.ROOT, "include", "tecdsa_b200.h")]
    if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in deps):
        subprocess.check_call(["g++", "-O1", "-w", "-I", HERE, "-I", entry.CSRC, "-shared", "-fPIC", "-o", so, src])
    lib = ctypes.CDLL(so)
    V = ctypes.c_void_p
    lib.h_field_name.restype = ctypes.c_char_p
    lib.h_run.argtypes = [ctypes.c_int, V, ctypes.c_int] + [V] * 7
    lib.h_init()
    return lib


class Arena:
    """The arena of csrc/gg20.cu for U units over `sessions` two-signer sessions (units 2s and 2s + 1, peer = u ^ 1)."""

    def __init__(self, hs, sessions):
        self.hs, self.U = hs, 2 * sessions
        n = hs.h_field_count()
        self.size = {hs.h_field_name(f).decode(): hs.h_field_size(f) for f in range(n)}
        self.off, acc = {}, 0
        for f in range(n):
            name = hs.h_field_name(f).decode()
            self.off[name] = acc
            acc += self.size[name]
        self.mem = np.zeros(acc * self.U, np.uint32)
        U = self.U
        self.peer = np.arange(U, dtype=np.uint32) ^ 1
        self.keyset = (np.arange(U) // 2).astype(np.uint32)            # one key set per session: ypk carries each session's y
        self.row_own = (np.arange(U) % 2).astype(np.uint32)
        self.row_peer = self.row_own ^ 1
        self.status = np.zeros(U, np.uint8)
        self.ypk = np.zeros((sessions, 16), np.uint32)
        rng = random.Random(0x5E55)
        self.tables = [np.array([rng.getrandbits(32) | 1 for _ in range(2 * k)], np.uint32) for k in KEY_SIZE]
        self._tp = (ctypes.c_void_p * len(KEY_SIZE))(*[t.ctypes.data for t in self.tables])

    def f(self, name, u):
        o_, s = self.off[name], self.size[name]
        return self.mem[o_ * self.U + u * s: o_ * self.U + (u + 1) * s]

    def flags(self, u):
        return self.f("FLAGS", u).view(np.uint8)

    def run(self, kernel):
        P = lambda a: a.ctypes.data
        assert self.hs.h_run(kernel, P(self.mem), self.U, ctypes.cast(self._tp, ctypes.c_void_p), P(self.ypk), P(self.row_own),
                             P(self.row_peer), P(self.peer), P(self.keyset), P(self.status)) == 0


# ------------------------------------------------------------------------------------------------ check kernels
@pytest.mark.parametrize("kernel,byte", [(R3_CHECK, PED), (R5_CHECK, PDL_BYTE), (R6_CHECK, HEG)])
def test_check_kernels_write_only_the_own_verdict(hs, kernel, byte):
    """one thread per unit, each writes byte `byte` of its own unit and nothing else of the FLAGS field (the peer's copy of the
    check, formerly byte + 1, is gone); garbage proofs are rejected"""
    A = Arena(hs, 3)
    rng = np.random.default_rng(1)
    for name in ("PED", "T", "HEG", "SI", "R", "RD", "PU1", "PU2", "PU3", "VE0", "VU20", "VU30", "PS1"):
        for u in range(A.U):
            A.f(name, u)[:] = rng.integers(0, 2 ** 32, A.size[name], dtype=np.uint32)
    for u in range(A.U):
        A.flags(u)[:] = 0xA5
    A.run(kernel)
    for u in range(A.U):
        fl = A.flags(u).copy()
        assert fl[byte] == 0, (u, fl)
        fl[byte] = 0xA5
        assert (fl == 0xA5).all(), (u, byte, fl)
    assert not A.status.any()


# ------------------------------------------------------------------------------------------------ finish kernels
def _honest_arena(hs, sessions=3, seed=7):
    """every verdict true, R_dash and S sums right, delta sums non-zero: all statuses 0 after the three finish kernels"""
    A = Arena(hs, sessions)
    rng = random.Random(seed)
    for s in range(sessions):
        R = o.pt_mul(o.G, rng.randrange(1, o.Q))
        rd0 = o.pt_mul(o.G, rng.randrange(1, o.Q))
        rds = [rd0, o.pt_add(o.G, o.pt_neg(rd0))]                  # R_dash_0 + R_dash_1 == G
        for p in range(2):
            u = 2 * s + p
            A.f("DELTA", u)[:] = L(rng.randrange(1, o.Q // 2), 8)
            A.f("R", u)[:] = pt16(R)
            A.f("RD", u)[:] = pt16(rds[p])
            A.f("SIGMA", u)[:] = L(rng.randrange(1, o.Q), 8)
            A.f("T", u)[:] = pt16(o.pt_mul(o.G, rng.randrange(1, o.Q)))
            rnd = A.f("RND", u)
            for off in (RND_L, RND_HEG_S1, RND_HEG_S2):
                rnd[off:off + 8] = L(rng.randrange(1, o.Q), 8)
            fl = A.flags(u)
            fl[PED] = fl[PDL_BYTE] = fl[HEG] = 1
            fl[PED + 1] = fl[PDL_BYTE + 1] = fl[HEG + 1] = 0         # stale bytes of the removed second checks: never read
    return A


def _finish(A):
    """r3 -> r5 -> r6 finish kernels; y of each session is set after r5 has written S, so that only injected failures fail"""
    A.run(R3_FINISH)
    A.run(R5_FINISH)
    for s in range(A.U // 2):
        if A.ypk[s].any():
            continue
        A.ypk[s] = pt16(o.pt_add(from16(A.f("SI", 2 * s)), from16(A.f("SI", 2 * s + 1))))
    A.run(R6)


def _two_check_status(A, own, pre_status, bad_rd_sum):
    """the status of every unit in the version where each unit checks both proofs of its session itself: verdict (u, j) is
    own[src][kind] with src = u for j = 0 and the peer for j = 1; the first failing check of a unit sets its status"""
    out = []
    for u in range(A.U):
        pu = u ^ 1
        st = pre_status[u]

        def fail(code):
            nonlocal st
            st = st or code
        if not (own[u][PED] and own[pu][PED]):
            fail(PROOF)
        if not (own[u][PDL_BYTE] and own[pu][PDL_BYTE]):
            fail(PDL)
        if bad_rd_sum[u // 2]:
            fail(PHASE5)
        if not (own[u][HEG] and own[pu][HEG]):
            fail(PHASE6)
        out.append(st)
    return out


def test_honest_sessions_pass(hs):
    A = _honest_arena(hs)
    _finish(A)
    assert list(A.status) == [OK] * A.U


@pytest.mark.parametrize("byte,code", [(PED, PROOF), (PDL_BYTE, PDL), (HEG, PHASE6)])
def test_one_false_verdict_fails_both_units_of_its_session(hs, byte, code):
    """for every session position and every unit: a verdict false on that unit alone fails it and its peer with the proof's
    code, as in the two-check version, and leaves the other sessions alone"""
    for v in range(6):
        A = _honest_arena(hs)
        A.flags(v)[byte] = 0
        own = [dict((b, int(A.flags(u)[b])) for b in (PED, PDL_BYTE, HEG)) for u in range(A.U)]
        want = _two_check_status(A, own, [0] * A.U, [False] * 3)
        _finish(A)
        assert list(A.status) == want, (v, byte, list(A.status))
        assert [u for u in range(A.U) if A.status[u]] == sorted([v, v ^ 1]) and set(A.status[[v, v ^ 1]]) == {code}


def test_status_precedence_is_unchanged(hs):
    """several failures at once: each unit keeps the first one in round order, an earlier round's status included"""
    rng = random.Random(11)
    for trial in range(12):
        A = _honest_arena(hs, seed=100 + trial)
        pre = [rng.choice([0, 0, 0, INVALID_KEY]) for _ in range(A.U)]
        A.status[:] = pre
        for u in range(A.U):
            for b in (PED, PDL_BYTE, HEG):
                if rng.random() < 0.2:
                    A.flags(u)[b] = 0
        bad_rd = [rng.random() < 0.3 for _ in range(3)]
        for s, bad in enumerate(bad_rd):
            if bad:                                                   # R_dash_0 + R_dash_1 != G
                A.f("RD", 2 * s)[:] = pt16(o.pt_mul(o.G, 5))
        own = [dict((b, int(A.flags(u)[b])) for b in (PED, PDL_BYTE, HEG)) for u in range(A.U)]
        want = _two_check_status(A, own, pre, bad_rd)
        _finish(A)
        assert list(A.status) == want, (trial, list(A.status), want)


# ------------------------------------------------------------------------------------------------ R symmetry
def _r4(hs, cases):
    """gg20_r3_finish (delta sum -> DINV) then gg20_r4_pre on one session per case; returns the R of both units"""
    A = Arena(hs, len(cases))
    for s, (g0, g1, d0, d1, k, alpha) in enumerate(cases):
        for p, (g, d) in enumerate(((g0, d0), (g1, d1))):
            u = 2 * s + p
            A.f("GG", u)[:] = pt16(g)
            A.f("DELTA", u)[:] = L(d, 8)
            rnd = A.f("RND", u)
            rnd[RND_K:RND_K + 8] = L(k[p], 8)
            rnd[RND_PDL_ALPHA:RND_PDL_ALPHA + 24] = L(alpha[p], 24)
    A.run(R3_FINISH)
    A.run(R4_PRE)
    return [(A.f("R", 2 * s).copy(), A.f("R", 2 * s + 1).copy()) for s in range(len(cases))]


def test_R_is_bit_identical_on_both_units(hs):
    rng = random.Random(0xA11)
    sc = lambda: rng.randrange(1, o.Q)
    g = o.pt_mul(o.G, sc())
    cases = []
    for _ in range(3):                                                # generic sessions
        cases.append((o.pt_mul(o.G, sc()), o.pt_mul(o.G, sc()), sc(), sc(), (sc(), sc()), (sc(), sc())))
    d = sc()
    cases += [
        (g, g, sc(), sc(), (sc(), sc()), (sc(), sc())),                     # Gamma_u == Gamma_peer: the doubling branch
        (g, o.pt_neg(g), sc(), sc(), (sc(), sc()), (sc(), sc())),           # Gamma_u == -Gamma_peer: R at infinity
        (None, g, sc(), sc(), (sc(), sc()), (sc(), sc())),                  # gamma = 0 on one unit
        (o.pt_mul(o.G, sc()), o.pt_mul(o.G, sc()), d, o.Q - d, (sc(), sc()), (sc(), sc())),   # delta sum 0: R at infinity
        (o.pt_mul(o.G, sc()), o.pt_mul(o.G, sc()), sc(), sc(), (0, sc()), (sc(), sc())),      # k = 0 on one unit: R_dash at infinity
        (o.pt_mul(o.G, sc()), o.pt_mul(o.G, sc()), sc(), sc(), (0, 0), (sc(), sc())),         # k = 0 on both units
        (o.pt_mul(o.G, sc()), o.pt_mul(o.G, sc()), sc(), sc(), (sc(), sc()), (0, o.Q)),       # alpha = 0 and alpha = q
        (o.pt_mul(o.G, sc()), o.pt_mul(o.G, sc()), sc(), sc(), (0, sc()), (o.Q * 7, 0)),      # k = 0 and alpha = 0 mod q together
    ]
    got = _r4(hs, cases)
    for i, ((g0, g1, d0, d1, _, _), (r0, r1)) in enumerate(zip(cases, got)):
        assert np.array_equal(r0, r1), i
        ds = (d0 + d1) % o.Q
        want = None if ds == 0 else o.pt_mul(o.pt_add(g0, g1), pow(ds, -1, o.Q))
        assert from16(r0) == want, i
