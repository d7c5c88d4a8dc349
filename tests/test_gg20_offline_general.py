"""CPU tests of the GG20 offline stage for any signing set as one call (tecdsa_gg20_offline_general_batch): the per-element,
per-pair and per-session kernels of csrc/gg20_general_kernels.cuh on the host harness against the oracle — Lagrange coefficients,
w_i and g_w_vec for signing sets of 2..16 out of up to 64 parties, the delta / sigma sums and the round-2 key check, the session
sums of delta, R_dash and S, and the session stop rule with failures injected in every round — plus the two new exports in the
header, the package and the Rust FFI."""
import ctypes
import os
import random
import subprocess

import numpy as np
import pytest

import __graft_entry__ as entry
from oracle import gg20_general_oracle as gen
from oracle import gg20_oracle as o

Q, G = o.Q, o.G
HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "host_harness")
OK, INVALID_KEY, PDL, PHASE5, PHASE6, PROOF, COMMIT = 0, 2, 6, 7, 8, 10, 11


def L(v, k):
    return np.frombuffer(int(v).to_bytes(4 * k, "little"), dtype=np.uint32).copy()


def I(a):
    return int.from_bytes(np.ascontiguousarray(a).tobytes(), "little")


def P_(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def pt16(p):
    return np.zeros(16, np.uint32) if p is None else np.concatenate([L(p[0], 8), L(p[1], 8)])


def from16(a):
    return None if not a.any() else (I(a[:8]), I(a[8:16]))


def rows(vals, k):
    return np.stack([L(v, k) for v in vals]) if vals else np.zeros((0, k), np.uint32)


@pytest.fixture(scope="module")
def hg():
    so = os.path.join(HERE, "libgg20_general_host.so")
    src = os.path.join(HERE, "gg20_general_harness.cpp")
    deps = [src] + [os.path.join(entry.CSRC, f) for f in os.listdir(entry.CSRC) if f.endswith((".cuh", ".h"))] + \
           [os.path.join(entry.ROOT, "include", "tecdsa_b200.h")]
    if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in deps):
        subprocess.check_call(["g++", "-O1", "-w", "-I", HERE, "-I", entry.CSRC, "-shared", "-fPIC", "-o", so, src])
    lib = ctypes.CDLL(so)
    V, I_ = ctypes.c_void_p, ctypes.c_int
    lib.h_index.argtypes = [V, I_, I_, I_] + [V] * 6
    lib.h_lagrange.argtypes = [V, I_, I_, V, V, V, V, I_]
    lib.h_msgb_status.argtypes = [V, I_, I_, I_, V, I_]
    lib.h_round1.argtypes = [I_, I_, V, V]
    lib.h_round2.argtypes = [I_, I_] + [V] * 11
    lib.h_round3.argtypes = [I_, V, V, V, V, I_]
    lib.h_round5.argtypes = [I_, I_, V, V, V, I_]
    lib.h_round6.argtypes = [I_, V, V, V, V, V, I_]
    lib.h_round_end.argtypes = [I_, V, V, V, I_]
    lib.h_finish.argtypes = [I_] + [V] * 10 + [I_]
    lib.h_init()
    return lib


def _ind(p, j):
    return j if j < p else j + 1


def test_index_tables(hg):
    """key rows, statement rows and the pair tables follow the convention of gg20_general.py (pair j * E + u: u towards ind(p, j))"""
    rng = random.Random(0x1D)
    T, P, n = 3, 5, 4
    d = [[rng.randrange(2)] + rng.sample(range(P), T) for _ in range(n)]
    E, NP = n * T, (T - 1) * n * T
    sess = np.array(d, np.uint32)
    out = [np.zeros(x, np.uint32) for x in (E, P * E, P * E, 2 * NP, 2 * NP, 2 * NP)]
    hg.h_index(P_(sess), T, P, E, *[P_(a) for a in out])
    row, st_row, st_elem, me, peer, row_peer = out
    own = [d[u // T][0] * P + d[u // T][1 + u % T] for u in range(E)]
    assert list(row) == own
    assert list(st_row) == [d[t % E // T][0] * P + t // E for t in range(P * E)] and list(st_elem) == [t % E for t in range(P * E)]
    for t in range(2 * NP):
        q = t % NP
        u, j = q % E, q // E
        v = u - u % T + _ind(u % T, j)
        assert (me[t], peer[t], row_peer[t]) == (u, v, own[v])


def test_lagrange_w_and_g_w_match_oracle(hg):
    """SignKeys::create / g_w_vec for random signing sets of 2..16 signers out of up to 64 parties, every session its own key set"""
    rng = random.Random(0x1A6)
    for T in range(2, 17):
        P = rng.randrange(T, 65)
        n = 2
        d = [[s] + rng.sample(range(P), T) for s in range(n)]
        xi = [rng.randrange(Q) for _ in range(n * P)]
        used = {s * P + i for s in range(n) for i in d[s][1:]}
        pk = [o.pt_mul(G, x) if r in used else None for r, x in enumerate(xi)]
        sess, XI, PK = np.array(d, np.uint32), rows(xi, 8), np.stack([pt16(p) for p in pk])
        E = n * T
        w, gw = np.zeros((E, 8), np.uint32), np.zeros((E, 16), np.uint32)
        hg.h_lagrange(P_(sess), T, P, P_(XI), P_(PK), P_(w), P_(gw), E)
        for u in range(E):
            s, p = divmod(u, T)
            l_s = d[s][1:]
            lam = o.lagrange_at_zero(l_s[p], l_s)
            r = s * P + l_s[p]
            assert I(w[u]) == lam * xi[r] % Q, (T, P, u)
            assert from16(gw[u]) == o.pt_mul(pk[r], lam), (T, P, u)
        # the Lagrange-weighted shares of a real sharing interpolate the secret: sum w_i = f(0)
        coef = [rng.randrange(1, Q) for _ in range(T)]
        f = lambda x: sum(c * pow(x, k, Q) for k, c in enumerate(coef)) % Q
        XI2 = rows([f(r % P + 1) for r in range(n * P)], 8)
        hg.h_lagrange(P_(sess), T, P, P_(XI2), P_(PK), P_(w), P_(gw), E)
        for s in range(n):
            assert sum(I(w[s * T + p]) for p in range(T)) % Q == coef[0]


def _pairs(rng, T, n):
    """random per-pair MtA results in the kernel layout (2 halves x [T-1][E]) and the receiving view of the oracle:
    recv[v][b] = the pair in which b sent to v"""
    E = n * T
    NP = (T - 1) * E
    pair = lambda u, j: j * E + u
    back = {}
    for u in range(E):
        for j in range(T - 1):
            back[(u, u - u % T + _ind(u % T, j))] = pair(u, j)
    return E, NP, back


def test_round2_sums_and_key_check(hg):
    """delta_i = k gamma + sum alpha + sum beta and sigma_i = k w + sum mu + sum nu over the pairs (party_i.rs:591-618), and the
    MessageB(w) key check against g_w_vec[sender] (rounds.rs:281): a wrong key fails its receiver only"""
    rng = random.Random(0x2D)
    for T in (2, 3, 5):
        n = 3
        E, NP, back = _pairs(rng, T, n)
        k, gam, w = ([rng.randrange(1, Q) for _ in range(E)] for _ in range(3))
        gw_s = [rng.randrange(1, Q) for _ in range(E)]
        gw = [o.pt_mul(G, x) for x in gw_s]
        alpha = [rng.randrange(Q) for _ in range(2 * NP)]
        beta = [rng.randrange(Q) for _ in range(2 * NP)]
        bp = np.zeros((2 * NP, 40), np.uint32)
        for (b, v), t in back.items():
            bp[NP + t, :16] = pt16(gw[b])
        st_a = np.zeros(2 * NP, np.uint8)
        bad_t = back[(1, 0)]                          # element 1 sends element 0 a MessageB(w) under a wrong key
        bp[NP + bad_t, :16] = pt16(o.pt_mul(G, gw_s[1] + 1))
        st_a[back[(E - 1, E - 2)]] = 2               # element E-2 fails get_alpha on what element E-1 sent it
        delta, sigma, cand = np.zeros((E, 8), np.uint32), np.zeros((E, 8), np.uint32), np.zeros(E, np.uint8)
        args = [rows(alpha, 8), rows(beta, 8), bp, np.stack([pt16(p) for p in gw]), rows(k, 8), rows(gam, 8), rows(w, 8)]
        hg.h_round2(T, E, P_(st_a), *[P_(a) for a in args], P_(delta), P_(sigma), P_(cand))
        for v in range(E):
            ins = [back[(v - v % T + _ind(v % T, j), v)] for j in range(T - 1)]
            outs = [j * E + v for j in range(T - 1)]
            assert I(delta[v]) == (k[v] * gam[v] + sum(alpha[t] for t in ins) + sum(beta[t] for t in outs)) % Q
            assert I(sigma[v]) == (k[v] * w[v] + sum(alpha[NP + t] for t in ins) + sum(beta[NP + t] for t in outs)) % Q
            assert cand[v] == (INVALID_KEY if v in (0, E - 2) else OK), (T, v)


def test_round1_and_msgb_status(hg):
    """one failed range proof of a sender's MessageA makes every MessageB that answers it fail, and round 1 stops the
    answering elements (mod.rs:123-131 -> InvalidKey)"""
    T, n, P = 3, 2, 4
    E, NP = n * T, (T - 1) * n * T
    pst = np.zeros(P * E, np.uint8)
    pst[2 * E + 4] = 5                            # statement 2 of element 4's MessageA
    pair_st = np.full(2 * NP, 255, np.uint8)
    hg.h_msgb_status(P_(pst), P, T, E, P_(pair_st), NP)
    for t in range(2 * NP):
        q = t % NP
        u, j = q % E, q // E
        assert pair_st[t] == (5 if u - u % T + _ind(u % T, j) == 4 else 0)
    cand = np.zeros(E, np.uint8)
    hg.h_round1(T, E, P_(pair_st), P_(cand))
    assert list(cand) == [0, 0, 0, INVALID_KEY, 0, INVALID_KEY]


def test_session_sums(hg):
    """round 3: sum delta and its inverse for every member, a failed Pedersen proof or delta = 0 stops the session; round 5: a
    failed PDL proof, else sum R_dash != G; round 6: a failed HomoElGamal proof or sum S != y"""
    rng = random.Random(0x5E55)
    T, n = 4, 4
    E = n * T
    delta = [rng.randrange(Q) for _ in range(E)]
    delta[T:2 * T] = [5, 7, Q - 12, 0]           # session 1 sums to zero
    ped = np.zeros(E, np.uint8)
    ped[2 * T + 3] = PROOF
    dinv, cand = np.zeros((E, 8), np.uint32), np.zeros(E, np.uint8)
    hg.h_round3(T, P_(rows(delta, 8)), P_(ped), P_(dinv), P_(cand), n)
    for s in range(n):
        tot = sum(delta[s * T:(s + 1) * T]) % Q
        bad = s in (1, 2)
        assert list(cand[s * T:(s + 1) * T]) == [PROOF if bad else OK] * T
        assert all(I(dinv[s * T + p]) == (0 if bad else pow(tot, -1, Q)) for p in range(T))
    # round 5: sessions whose R_dash sum to G, one tampered, one with a failed PDL proof
    Rd = []
    for s in range(n):
        xs = [rng.randrange(1, Q) for _ in range(T - 1)]
        xs.append((1 - sum(xs)) % Q)
        Rd += [o.pt_mul(G, x) for x in xs]
    Rd[T] = o.pt_mul(G, 3)
    pdl = np.zeros((T - 1) * E, np.uint8)
    pdl[1 * E + 2 * T + 1] = PDL
    hg.h_round5(T, E, P_(pdl), P_(np.stack([pt16(p) for p in Rd])), P_(cand), n)
    assert [cand[s * T] for s in range(n)] == [OK, PHASE5, PDL, OK] and all(cand[s * T + p] == cand[s * T] for s in range(n) for p in range(T))
    # round 6: S_i = s_i G with sum s_i = the key set's secret
    ys = [rng.randrange(1, Q) for _ in range(2)]
    d = np.array([[s % 2] + list(range(T)) for s in range(n)], np.uint32)
    S = []
    for s in range(n):
        xs = [rng.randrange(1, Q) for _ in range(T - 1)]
        xs.append((ys[s % 2] - sum(xs)) % Q)
        S += [o.pt_mul(G, x) for x in xs]
    S[3 * T + 2] = o.pt_mul(G, 9)
    heg = np.zeros(E, np.uint8)
    heg[T] = PROOF
    hg.h_round6(T, P_(d), P_(heg), P_(np.stack([pt16(p) for p in S])), P_(np.stack([pt16(o.pt_mul(G, y)) for y in ys])), P_(cand), n)
    assert [cand[s * T] for s in range(n)] == [OK, PHASE6, OK, PHASE6]


def test_stop_rule_with_failures_in_every_round(hg):
    """The status assembly over six rounds against the Python driver's rule (gg20_general.py: `fail` records an error only for an
    element without one in a session not yet stopped; `end_round` stops every session with an error): a session stops at its
    first failing round, later failures of its members are not recorded, other sessions are untouched; finish zeroes the
    outputs of incomplete sessions"""
    rng = random.Random(0x570)
    T, n = 3, 8
    E = n * T
    codes = [INVALID_KEY, INVALID_KEY, PROOF, COMMIT, PDL, PHASE6]
    plan = {1: (0, [0]), 2: (1, [1, 2]), 3: (2, [0, 1, 2]), 4: (3, [2]), 5: (4, [0, 1, 2]), 6: (5, [1])}   # session -> (round, positions)
    status, stopped = np.zeros(E, np.uint8), np.zeros(n, np.uint8)
    want, stop = [0] * E, set()
    for rnd in range(6):
        cand = np.zeros(E, np.uint8)
        for s, (r, ps) in plan.items():
            if r <= rnd:                                            # a failed check keeps failing in later rounds
                for p in ps:
                    cand[s * T + p] = codes[rnd]
        if rnd == 5:
            cand[7 * T + 1] = PHASE6                                 # session 7 fails only in the last round
        hg.h_round_end(T, P_(cand), P_(status), P_(stopped), n)
        for u in range(E):
            if cand[u] and not want[u] and u // T not in stop:
                want[u] = int(cand[u])
        stop.update(u // T for u in range(E) if want[u])
        assert list(status) == want and list(stopped) == [int(s in stop) for s in range(n)]
    assert [status[s * T:(s + 1) * T].tolist() for s in (1, 2, 3)] == [[INVALID_KEY, 0, 0], [0, INVALID_KEY, INVALID_KEY], [PROOF] * 3]
    R, sg, Tp = (np.array([[rng.randrange(1, 2 ** 32) for _ in range(k)] for _ in range(E)], np.uint32) for k in (16, 8, 16))
    outs = [np.full(E, 255, np.uint8), np.full((E, 16), 7, np.uint32), np.full((E, 8), 7, np.uint32), np.full((E, 16), 7, np.uint32), np.full(n, 9, np.uint8)]
    hg.h_finish(T, P_(status), P_(stopped), P_(R), P_(sg), P_(Tp), *[P_(a) for a in outs], E)
    assert list(outs[0]) == list(status) and list(outs[4]) == [1, 0, 0, 0, 0, 0, 0, 0]
    for u in range(E):
        ok = u // T == 0
        assert (outs[1][u] == (R[u] if ok else 0)).all() and (outs[2][u] == (sg[u] if ok else 0)).all() and (outs[3][u] == (Tp[u] if ok else 0)).all()


def test_new_exports_in_header_package_and_ffi(pkg):
    import re
    hdr = open(os.path.join(entry.ROOT, "include", "tecdsa_b200.h")).read()
    ffi = open(os.path.join(entry.ROOT, "bindings", "rust", "src", "ffi.rs")).read()
    for name in ("tecdsa_keys_upload_parties", "tecdsa_gg20_offline_general_batch"):
        assert re.search(rf"\b{name}\s*\(", hdr) and name in pkg.EXPORTS and f"pub fn {name}(" in ffi
    for struct in ("tecdsa_offline_general_in", "tecdsa_offline_general_out"):
        assert f"pub struct {struct}" in ffi
    from mpecdsa_b200 import gg20_general
    assert [f for f, _ in gg20_general._GeneralIn._fields_] == re.findall(r"const uint32_t\* (\w+);", hdr.split("tecdsa_offline_general_in;")[0].split("typedef struct {")[-1])
