"""CPU-only: the seeded sampler.  The ChaCha20 restatement of oracle/seeded_sampling.py against RFC 8439 and `cryptography`; the
product's device code (csrc/chacha20.cuh, csrc/sampler.cuh) compiled for the host through tests/host_harness/sampler_harness.cpp
against that oracle, value by value and for the whole randomness record of an offline unit; and the host bookkeeping of
`gg20_general.sample_rnd` with `Engine.sample` stood in by the oracle (the technique of tests/test_host_drivers_cpu.py)."""
import ctypes
import math
import os
import random
import subprocess

import numpy as np
import pytest

import __graft_entry__ as entry
from oracle import gg20_general_oracle as gen
from oracle import gg20_oracle as o
from oracle import seeded_sampling as ss
from tests import test_gg20_general as tg
from tests.golden import fixtures

HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "host_harness")
BITS, BELOW, UNIT, RANGE1, SCALAR = range(5)
KIND = {BITS: "bits", BELOW: "below", UNIT: "unit", RANGE1: "range1", SCALAR: "scalar"}
Q = o.Q
SEED = bytes(range(100, 132))


@pytest.fixture(scope="module")
def h():
    so = os.path.join(HERE, "libsampler_host.so")
    src = os.path.join(HERE, "sampler_harness.cpp")
    deps = [src] + [os.path.join(entry.CSRC, f) for f in os.listdir(entry.CSRC) if f.endswith((".cuh", ".h"))] + \
           [os.path.join(entry.ROOT, "include", "tecdsa_b200.h")]
    if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in deps):
        subprocess.check_call(["g++", "-O1", "-w", "-I", HERE, "-I", entry.CSRC, "-shared", "-fPIC", "-o", so, src])
    lib = ctypes.CDLL(so)
    V, U32, U64, I = ctypes.c_void_p, ctypes.c_uint32, ctypes.c_uint64, ctypes.c_int
    lib.h_chacha_block.argtypes = [V, V, U32, U32, U32, U32]
    lib.h_sample.argtypes = [V, U32, U64, I, V, I, V, I, I, U32, V]
    lib.h_gg20_sample_bounds.argtypes = [V, V, V, I]
    lib.h_gg20_sample_field.argtypes = [V, U64, I, U32, U32, U32, V, V, V, V, U32]
    lib.h_gg20_sample_unit.argtypes = [V, U64, U32, U32, U32, V, V, V, V, U32]
    return lib


def L(v, k):
    return np.frombuffer(int(v).to_bytes(4 * k, "little"), dtype=np.uint32).copy()


def I(a):
    return int.from_bytes(np.ascontiguousarray(a).tobytes(), "little")


def P(a):
    return None if a is None else a.ctypes.data_as(ctypes.c_void_p)


def _key(seed):
    return np.frombuffer(seed, dtype="<u4").copy()


def dev_sample(h, seed, stream, ident, kind, limbs, bound=0, bits=0, cap=ss.ATTEMPTS):
    """smp::sample on the host harness -> (value, ok, attempts)"""
    out = np.full(limbs, 0xDEADBEEF, np.uint32)
    b = L(bound, limbs) if kind in (BELOW, UNIT, RANGE1) else None
    att = np.zeros(1, np.uint32)
    ok = h.h_sample(P(_key(seed)), stream, ident, kind, P(out), limbs, P(b), limbs, bits, cap, P(att))
    return I(out), bool(ok), int(att[0])


# ---- 1. the generator -------------------------------------------------------------------------------------------------------
RFC_8439_2_3_2 = bytes.fromhex(
    "10f1e7e4d13b5915500fdd1fa32071c4c7d1f4c733c068030422aa9ac3d46c4e"
    "d2826446079faa0914c2d705d98b02a2b5129cd1de164eb9cbd083e8a2503c4e")


def test_chacha20_block_is_rfc_8439(h):
    key, nonce = bytes(range(32)), bytes.fromhex("000000090000004a00000000")
    assert ss.chacha20_block(key, 1, nonce) == RFC_8439_2_3_2
    out = np.zeros(16, np.uint32)
    h.h_chacha_block(P(out), P(_key(key)), 1, 0x09000000, 0x4A000000, 0)
    assert out.tobytes() == RFC_8439_2_3_2


def test_chacha20_keystream_equals_cryptography(h):
    ciphers = pytest.importorskip("cryptography.hazmat.primitives.ciphers")
    rng = random.Random(0xC4AC4A)
    for _ in range(24):
        key, nonce, counter = rng.randbytes(32), rng.randbytes(12), rng.choice([0, 1, 7, 2 ** 31, 2 ** 32 - 9])
        enc = ciphers.Cipher(ciphers.algorithms.ChaCha20(key, counter.to_bytes(4, "little") + nonce), mode=None).encryptor()
        want = enc.update(bytes(64 * 5))
        assert b"".join(ss.chacha20_block(key, counter + b, nonce) for b in range(5)) == want
        n = [int.from_bytes(nonce[4 * i:4 * i + 4], "little") for i in range(3)]
        out = np.zeros(16, np.uint32)
        for b in range(5):
            h.h_chacha_block(P(out), P(_key(key)), counter + b, *n)
            assert out.tobytes() == want[64 * b:64 * b + 64]


# ---- 2. every kind against the oracle ------------------------------------------------------------------------------------
def _smooth_modulus(bits):
    n, p = 1, 3
    while True:
        if all(p % d for d in range(3, int(p ** 0.5) + 1, 2)):
            if (n * p).bit_length() > bits:
                return n
            n *= p
        p += 2


@pytest.mark.parametrize("limbs", [8, 24, 64, 72, 88, 128])
def test_every_kind_equals_oracle(h, limbs):
    rng = random.Random(limbs)
    k = 32 * limbs - 7
    bounds = [2 ** k, 2 ** k + 1, 2 ** k - 1, 2 ** (32 * (limbs - 1)) + rng.getrandbits(32 * (limbs - 1)), 1, 2, 3, 4, 5,
              rng.getrandbits(32 * limbs) | (1 << (32 * limbs - 1)), 2 ** (32 * limbs) - 1, 2 ** 32, 2 ** 32 + 1, 2 ** 32 + 2,
              rng.getrandbits(32 * limbs - 40) * 2]
    rejected = {b: 0 for b in bounds}
    for kind in (BELOW, UNIT, RANGE1):
        for bi, bound in enumerate(bounds):
            for ident in (0, 1, 2 ** 32 + 5, 2 ** 64 - 1):
                got = dev_sample(h, SEED, 40 + kind, ident + bi if ident < 2 ** 63 else ident, kind, limbs, bound)
                want = ss.sample(SEED, 40 + kind, ident + bi if ident < 2 ** 63 else ident, KIND[kind], bound)
                assert got == want, (kind, hex(bound), ident)
                if want[1]:
                    lo, hi = (1, bound - 1) if kind == RANGE1 else (0, bound)
                    assert lo <= want[0] < hi and (kind != UNIT or math.gcd(want[0], bound) == 1)
                    rejected[bound] += want[2] - 1 if kind == BELOW else 0
    # 2^k and 2^k + 1 are drawn on k + 1 bits: about half of the candidates are rejected; 2^k - 1 on k bits: none
    for bound in (2 ** k, 2 ** k + 1):
        for ident in range(100, 116):
            want = ss.sample(SEED, 41, ident, "below", bound)
            assert dev_sample(h, SEED, 41, ident, BELOW, limbs, bound) == want
            rejected[bound] += want[2] - 1
    assert rejected[2 ** k] > 0 and rejected[2 ** k + 1] > 0 and rejected[2 ** k - 1] == 0
    # degenerate bounds: a status and a zero value, never a draw
    for kind, bad in ((BELOW, [0]), (UNIT, [0, 1]), (RANGE1, [0, 1, 2])):
        for bound in bad:
            assert dev_sample(h, SEED, 1, 1, kind, limbs, bound) == (0, False, 0) == ss.sample(SEED, 1, 1, KIND[kind], bound)
    for bits in (1, 31, 32, 33, 256, 32 * limbs - 1, 32 * limbs):
        assert dev_sample(h, SEED, 2, bits, BITS, limbs, bits=bits) == ss.sample(SEED, 2, bits, "bits", bits=bits)
    for bits in (0, 32 * limbs + 1):
        assert dev_sample(h, SEED, 2, 0, BITS, limbs, bits=bits)[:2] == (0, False)
    for ident in range(6):
        got = dev_sample(h, SEED, 0, ident, SCALAR, limbs)
        assert got == ss.sample(SEED, 0, ident, "scalar") and 0 < got[0] < Q
    # a bound as wide as the row, drawn into a narrower one: no value can be produced
    if limbs > 8:
        out, att = np.zeros(8, np.uint32), np.zeros(1, np.uint32)
        assert h.h_sample(P(_key(SEED)), 0, 0, BELOW, P(out), 8, P(L(bounds[0], limbs)), limbs, 0, 256, P(att)) == 0 and att[0] == 0
    assert dev_sample(h, SEED, 0, 0, SCALAR, 4)[:2] == (0, False)


def test_unit_group_of_a_smooth_modulus_and_the_attempt_cap(h):
    n = _smooth_modulus(2048)
    assert n % 2 == 1 and 2030 < n.bit_length() <= 2048
    attempts = []
    for ident in range(40):
        got = dev_sample(h, SEED, 7, ident, UNIT, 64, n)
        want = ss.sample(SEED, 7, ident, "unit", n)
        assert got == want and got[1] and math.gcd(got[0], n) == 1
        attempts.append(want[2])
    assert sum(attempts) > 3 * len(attempts)                         # most candidates are rejected
    # the cap: an element that needs more than N attempts gets the status and a zero value with cap N, its value with a larger cap
    ident = max(range(40), key=lambda i: attempts[i])
    need = attempts[ident]
    assert need > 8
    for cap in (1, 8, need - 1):
        assert dev_sample(h, SEED, 7, ident, UNIT, 64, n, cap=cap) == (0, False, cap) == ss.sample(SEED, 7, ident, "unit", n, cap=cap)
    assert dev_sample(h, SEED, 7, ident, UNIT, 64, n, cap=need) == ss.sample(SEED, 7, ident, "unit", n, cap=need)
    assert dev_sample(h, SEED, 7, ident, UNIT, 64, n, cap=need)[1]
    # even moduli: v and m both even is a rejection, an odd v under an even m is tested with the roles swapped
    for m in (2 ** 2047 + 2 ** 100, n * 2, 6, 2 ** 64):
        for ident in range(4):
            lim = 64 if m.bit_length() > 96 else 8
            got = dev_sample(h, SEED, 8, ident, UNIT, lim, m)
            assert got == ss.sample(SEED, 8, ident, "unit", m) and math.gcd(got[0], m) == 1


# ---- 3. the whole record ---------------------------------------------------------------------------------------------------
def _layout(pkg):
    """stream id -> (offset, limbs) of the randomness record, from the host layer's TECDSA_RND_* tables"""
    from mpecdsa_b200 import gg20
    lay = {gg20.RNDS[{"gamma_i": "gamma", "k_i": "k"}.get(name, name)]: v for name, v in gg20.RND.items()}
    for x in range(3):
        for part, (off, limbs) in enumerate(gg20.RND_ALICE_PARTS):
            lay[gg20.RNDS_ALICE + 4 * x + part] = (gg20.RND_ALICE + x * gg20.RND_ALICE_STRIDE + off, limbs)
    for name, v in zip(("pdl_alpha", "pdl_beta", "pdl_rho", "pdl_gamma"), gg20.RND_PDL_PARTS):
        lay[gg20.RNDS[name]] = v
    return lay


def _key_tables(h, keyset):
    n_tab = np.concatenate([L(lk.dk.p * lk.dk.q, 64) for lk in keyset])
    nt_tab = np.concatenate([L(lk.h1_h2_n_tilde_vec[lk.i - 1].N, 64) for lk in keyset])
    qnt, q3nt = np.zeros(3 * 72, np.uint32), np.zeros(3 * 88, np.uint32)
    h.h_gg20_sample_bounds(P(nt_tab), P(qnt), P(q3nt), 3)
    for r, lk in enumerate(keyset):
        nt = lk.h1_h2_n_tilde_vec[lk.i - 1].N
        assert I(qnt[72 * r:72 * r + 72]) == Q * nt and I(q3nt[88 * r:88 * r + 88]) == Q ** 3 * nt
    return n_tab, qnt, q3nt


def test_record_equals_oracle_for_every_key_and_signer_pair(h, pkg):
    from mpecdsa_b200 import gg20
    keysets = fixtures.load_all_keysets() + fixtures.load_edge_keysets()
    assert any((lk.dk.p * lk.dk.q).bit_length() == 2047 for ks in keysets for lk in ks)
    unit = 2 ** 40
    for keyset in keysets:
        n_tab, qnt, q3nt = _key_tables(h, keyset)
        for a in range(3):
            for b in range(3):
                if a == b:
                    continue
                s_l, keys = [a + 1, b + 1], [keyset[a], keyset[b]]
                for pos, (own, peer) in enumerate(((a, b), (b, a))):
                    unit += 1
                    rec = np.full(gg20.RND_LIMBS, 0xDEADBEEF, np.uint32)
                    assert h.h_gg20_sample_unit(P(_key(SEED)), unit, own, peer, 0, P(n_tab), P(qnt), P(q3nt), P(rec), ss.ATTEMPTS) == 0
                    want = ss.sample_unit_seeded(SEED, unit, keys, s_l, pos)
                    assert (rec == gg20.pack_randomness([want])[0]).all(), (s_l, pos)
                    # every field inside its reference range
                    n_own, n_peer = keys[pos].dk.p * keys[pos].dk.q, keys[1 - pos].dk.p * keys[1 - pos].dk.q
                    nt_peer = keys[pos].h1_h2_n_tilde_vec[peer].N
                    for name in ("gamma_i", "k_i", "nonce_gamma_b", "nonce_gamma_beta", "nonce_w_b", "nonce_w_beta", "l", "ped_s1", "ped_s2", "heg_s1", "heg_s2"):
                        assert 0 < getattr(want, name) < Q
                    assert want.blind < 2 ** 256 and want.r_k < n_own
                    for x, (al, be, ga, rho) in enumerate(want.alice):
                        nt = keyset[x].h1_h2_n_tilde_vec[x].N
                        assert al < Q ** 3 and be < n_own and math.gcd(be, n_own) == 1 and ga < Q ** 3 * nt and rho < Q * nt
                    assert max(want.beta_tag_gamma, want.r_gamma, want.beta_tag_w, want.r_w) < n_peer
                    assert want.pdl[0] < Q ** 3 and 1 <= want.pdl[1] < n_own - 1 and want.pdl[2] < Q * nt_peer and want.pdl[3] < Q ** 3 * nt_peer


def test_fields_cover_the_record_exactly_once(h, pkg):
    from mpecdsa_b200 import gg20
    lay = _layout(pkg)
    assert sorted(lay) == list(range(33))
    keyset = fixtures.load_keyset(0)
    n_tab, qnt, q3nt = _key_tables(h, keyset)
    written = np.zeros(gg20.RND_LIMBS, int)
    for f in range(33):
        rec = np.full(gg20.RND_LIMBS, 0xDEADBEEF, np.uint32)
        assert h.h_gg20_sample_field(P(_key(SEED)), 9, f, 1, 2, 0, P(n_tab), P(qnt), P(q3nt), P(rec), ss.ATTEMPTS) == 1
        touched = np.flatnonzero(rec != 0xDEADBEEF)
        off, limbs = lay[f]
        assert list(touched) == list(range(off, off + limbs)), f
        written[touched] += 1
    assert (written == 1).all()
    rec = np.full(gg20.RND_LIMBS, 0xDEADBEEF, np.uint32)
    assert h.h_gg20_sample_field(P(_key(SEED)), 9, 33, 1, 2, 0, P(n_tab), P(qnt), P(q3nt), P(rec), ss.ATTEMPTS) == 0 and (rec == 0xDEADBEEF).all()


# ---- 4. distinctness -------------------------------------------------------------------------------------------------------
def test_units_fields_and_seeds_are_independent_streams(h):
    keyset = fixtures.load_keyset(0)
    keys, s_l = [keyset[0], keyset[1]], [1, 2]
    a = ss.sample_unit_seeded(SEED, 10, keys, s_l, 0)
    b = ss.sample_unit_seeded(SEED, 11, keys, s_l, 0)
    c = ss.sample_unit_seeded(bytes(32), 10, keys, s_l, 0)
    scalars = ("gamma_i", "k_i", "nonce_gamma_b", "nonce_gamma_beta", "nonce_w_b", "nonce_w_beta", "l", "ped_s1", "ped_s2", "heg_s1", "heg_s2")
    assert len({getattr(r, f) for r in (a, b, c) for f in scalars}) == 3 * len(scalars)
    assert len({v for r in (a, b, c) for v in (r.r_k, r.beta_tag_gamma, r.r_gamma, r.beta_tag_w, r.r_w, r.pdl[1], *[t[1] for t in r.alice])}) == 3 * 9
    # first_unit shifts the element ids, it does not reseed: element 3 of a batch starting at 7 is element 10
    assert dev_sample(h, SEED, 1, 7 + 3, SCALAR, 8)[0] == a.k_i == ss.sample(SEED, 1, 10, "scalar")[0]


# ---- 5. gg20_general.sample_rnd: host bookkeeping with Engine.sample stood in by the oracle ------------------------------------
class _Keys:
    def __init__(self, rows):
        self.rows = rows

    def table(self, index, limbs):
        assert (index, limbs) in ((0, 64), (2, 64))
        return [lk.dk.p * lk.dk.q if index == 0 else lk.h1_h2_n_tilde_vec[lk.i - 1].N for lk in self.rows]


class _Engine:
    def __init__(self):
        self.used = set()

    def sample(self, kind, count, seed, stream=0, first_id=0, bound=None, bound_idx=None, bits=0, limbs=None):
        vals, st = [], np.zeros(count, np.uint8)
        for i in range(count):
            assert (stream, first_id + i) not in self.used, "a (stream, element id) pair drawn twice under one seed"
            self.used.add((stream, first_id + i))
            v, ok, _ = ss.sample(seed, stream, first_id + i, KIND[kind], 0 if bound is None else bound[i if bound_idx is None else bound_idx[i]], bits)
            vals.append(v); st[i] = 0 if ok else 13
        return vals, st


def _party_randomness(rnd, u, ttag):
    P1 = ttag - 1
    r = gen.PartyRandomness(gamma_i=rnd["gamma"][u], k_i=rnd["k"][u], blind=rnd["blind"][u], r_k=rnd["r_k"][u], alice=list(rnd["alice"][u]),
                            l=rnd["l"][u], ped_s1=rnd["ped_s1"][u], ped_s2=rnd["ped_s2"][u], heg_s1=rnd["heg_s1"][u], heg_s2=rnd["heg_s2"][u])
    for f in ("beta_tag_gamma", "r_gamma", "nonce_gamma_b", "nonce_gamma_beta", "beta_tag_w", "r_w", "nonce_w_b", "nonce_w_beta", "pdl"):
        setattr(r, f, [rnd[f][u * P1 + j] for j in range(P1)])
    return r


@pytest.mark.parametrize("case", ["t1n3_two", "t1n3_three", "t2n5_three"])
def test_sample_rnd_drives_the_general_oracle_to_completed_sessions(pkg, case):
    from mpecdsa_b200 import gg20_general
    keysets = fixtures.load_all_keysets()[:2]
    rng = random.Random(7)
    if case == "t2n5_three":
        key5 = tg._five_party_key(keysets, rng)
        rows = [lk for ks in keysets for lk in ks][:5]
        sessions = [([key5[i - 1] for i in s_l], s_l) for s_l in ([5, 2, 3], [1, 4, 2])]
        row_of = lambda lk, j: j
    else:
        rows = [lk for ks in keysets for lk in ks]
        lists = [(0, [1, 2]), (1, [3, 1]), (0, [2, 3])] if case == "t1n3_two" else [(0, [1, 2, 3]), (1, [3, 1, 2])]
        sessions = [([keysets[k][i - 1] for i in s_l], s_l) for k, s_l in lists]
        owner = {id(lk): k for k, ks in enumerate(keysets) for lk in ks}
        row_of = lambda lk, j: 3 * owner[id(lk)] + j
    ttag = len(sessions[0][1])
    key_rows = [row_of(lk, lk.i - 1) for keys, _ in sessions for lk in keys]
    all_rows = [[row_of(lk, j) for j in range(lk.n)] for keys, _ in sessions for lk in keys]
    eng = _Engine()
    rnd = gg20_general.sample_rnd(eng, _Keys(rows), ttag, key_rows, all_rows, seed=SEED)
    assert gg20_general.sample_rnd(_Engine(), _Keys(rows), ttag, key_rows, all_rows, seed=SEED) == rnd          # a pure function of the seed
    assert gg20_general.sample_rnd(_Engine(), _Keys(rows), ttag, key_rows, all_rows)["k"] != rnd["k"]           # seed=None: a fresh one
    u = 0
    for keys, s_l in sessions:
        pr = [_party_randomness(rnd, u + p, ttag) for p in range(ttag)]
        for p, (lk, r) in enumerate(zip(keys, pr)):
            n_own = lk.dk.p * lk.dk.q
            assert len(r.alice) == lk.n and all(math.gcd(t[1], n_own) == 1 and t[2] < Q ** 3 * lk.h1_h2_n_tilde_vec[x].N for x, t in enumerate(r.alice))
            for j in range(ttag - 1):
                peer = s_l[gen._ind(p, j)] - 1
                assert r.r_gamma[j] < lk.paillier_key_vec[peer].n and r.beta_tag_w[j] < lk.paillier_key_vec[peer].n
                assert 1 <= r.pdl[j][1] < n_own - 1 and r.pdl[j][3] < Q ** 3 * lk.h1_h2_n_tilde_vec[peer].N
        res = gen.offline_session(keys, s_l, pr)
        assert [x.status for x in res] == [0] * ttag and tg._signature_ok(res, keys[0].y_sum_s, rng)
        u += ttag
