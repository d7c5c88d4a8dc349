"""CPU tests of GG20 key generation as one call (tecdsa_gg20_keygen_batch): the party-by-party restatement tests/keygen_group.py
against the per-phase oracle functions and the algebra a key must satisfy (y = sum u_i G, pk_j = x_j G, any t + 1 shares interpolate
to sum u_i, a (2, 5) key signs), the group-level kernels of csrc/keygen_kernels.cuh on the host harness against the oracle (honest
inputs, every tampered field, status precedence), and the new export in the header, the package and the Rust FFI."""
import ctypes
import os
import random
import re
import subprocess

import numpy as np
import pytest

import __graft_entry__ as entry
from oracle import gg20_general_oracle as gen
from oracle import gg20_oracle as o
from oracle import keygen_oracle as kg
from tests import keygen_group as kgg
from tests.golden import fixtures

Q, G = o.Q, o.G
HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "host_harness")


def fixture_primes(n, offset=0):
    """Paillier primes of fixture rows offset.., N~ primes from the Paillier primes of rows 12.. (distinct keys, 2048-bit products)"""
    rows = [lk for ks in fixtures.load_all_keysets() for lk in ks]
    return [((rows[offset + i].dk.p, rows[offset + i].dk.q), (rows[12 + offset + i].dk.p, rows[12 + offset + i].dk.q)) for i in range(n)]


def group(t, n, seed, offset=0):
    rng = random.Random(seed)
    primes = fixture_primes(n, offset)
    rnd = [kgg.random_inputs(t, pr[1], rng) for pr in primes]
    return primes, rnd


# ------------------------------------------------------------------------------------------------ the oracle
def test_keygen_group_equals_per_phase_flow():
    """(1, 3): the group oracle's LocalKeys are the values of tests/test_keygen_oracle.py's three-party flow"""
    t, n = 1, 3
    primes, rnd = group(t, n, 0x6B01)
    keys, status, bad = kgg.keygen_group(t, n, primes, rnd)
    assert status == [0] * n and bad == [0] * n
    vss = [kg.vss_share(t, n, r["u"], r["coeffs"]) for r in rnd]
    for i, lk in enumerate(keys):
        assert lk.x_i == sum(vss[j][1][i] for j in range(n)) % Q
        assert lk.vss_commitments == vss[i][0].commitments
        (p, q), (pt, qt) = primes[i]
        nt, h1, h2, _, _ = kg.h1_h2_n_tilde(pt, qt, rnd[i]["h1"], rnd[i]["xhi"])
        assert (lk.h1_h2_n_tilde_vec[i].N, lk.h1_h2_n_tilde_vec[i].g, lk.h1_h2_n_tilde_vec[i].ni) == (nt, h1, h2)
        assert lk.paillier_key_vec[i].n == p * q and lk.dk.p == p
    assert kg.commitments_to_xi([v[0] for v in vss]) == keys[0].pk_vec


@pytest.mark.parametrize("t,n", [(1, 3), (2, 5), (3, 4), (1, 2)])
def test_keygen_group_key_algebra(t, n):
    primes, rnd = group(t, n, 0x6B00 + 16 * t + n)
    keys, status, bad = kgg.keygen_group(t, n, primes, rnd)
    assert status == [0] * n and bad == [0] * n
    secret = sum(r["u"] for r in rnd) % Q
    assert all(lk.y_sum_s == o.pt_mul(G, secret) for lk in keys)
    assert all(lk.pk_vec[j] == o.pt_mul(G, keys[j].x_i) for lk in keys for j in range(n))
    rng = random.Random(n)
    for _ in range(3):
        sub = rng.sample(range(n), t + 1)
        assert kgg.lagrange_at_zero([(j + 1, keys[j].x_i) for j in sub]) == secret


def test_keygen_group_failures():
    t, n = 1, 3
    primes, rnd = group(t, n, 0x6B10)
    # a 2046-bit Paillier modulus at party 2: every party rejects its broadcast
    bad_primes = list(primes)
    bad_primes[1] = ((primes[1][0][0] >> 2 | 1, primes[1][0][1]), primes[1][1])
    keys, status, bad = kgg.keygen_group(t, n, bad_primes, rnd)
    assert keys == [None] * n and status == [kgg.ST_INVALID_KEY] * n and bad == [0b010] * n
    # p = q at party 3
    bad_primes = list(primes)
    bad_primes[2] = ((primes[2][0][0], primes[2][0][0]), primes[2][1])
    assert kgg.keygen_group(t, n, bad_primes, rnd)[1:] == ([kgg.ST_INVALID_KEY] * n, [0b100] * n)
    # an xhi sharing a factor with phi(N~) at party 1: NOT_INVERTIBLE on that element alone
    bad_rnd = [dict(r) for r in rnd]
    bad_rnd[0]["xhi"] = 2 * (rnd[0]["xhi"] // 2)
    assert kgg.keygen_group(t, n, primes, bad_rnd)[1:] == ([kgg.ST_NOT_INVERTIBLE, 0, 0], [0, 0, 0])


def test_five_party_key_signs():
    """a (2, 5) key from the group oracle signs through the size-generic offline oracle; OpenSSL accepts the signature"""
    from cryptography.hazmat.primitives import hashes
    from cryptography.hazmat.primitives.asymmetric import ec, utils
    from tests import test_gg20_general as tg
    primes, rnd = group(2, 5, 0x6B25)
    keys, status, _ = kgg.keygen_group(2, 5, primes, rnd)
    assert status == [0] * 5
    rng = random.Random(0x6B26)
    s_l = [4, 1, 5]
    signers = [keys[i - 1] for i in s_l]
    srnd = [tg._party_randomness(rng, lk, [s_l[gen._ind(p, j)] - 1 for j in range(2)]) for p, lk in enumerate(signers)]
    res = gen.offline_session(signers, s_l, srnd)
    assert [x.status for x in res] == [0, 0, 0]
    m = rng.getrandbits(256) % Q
    r_, s_, _ = o.output_signature(res[0].R, [o.local_sig(x.k_i, m, x.R, x.sigma_i) for x in res])
    y = keys[0].y_sum_s
    pub = ec.EllipticCurvePublicNumbers(y[0], y[1], ec.SECP256K1()).public_key()
    pub.verify(utils.encode_dss_signature(r_, s_), m.to_bytes(32, "big"), ec.ECDSA(utils.Prehashed(hashes.SHA256())))


# ------------------------------------------------------------------------------------------------ kernels on the host harness
def L(v, k):
    return np.frombuffer(int(v).to_bytes(4 * k, "little"), dtype=np.uint32).copy()


def I(a):
    return int.from_bytes(np.ascontiguousarray(a).tobytes(), "little")


def P(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def pt16(p):
    return np.zeros(16, np.uint32) if p is None else np.concatenate([L(p[0], 8), L(p[1], 8)])


def from16(a):
    return None if not a.any() else (I(a[:8]), I(a[8:16]))


@pytest.fixture(scope="module")
def hk():
    so = os.path.join(HERE, "libkeygen_host.so")
    src = os.path.join(HERE, "keygen_harness.cpp")
    deps = [src] + [os.path.join(entry.CSRC, f) for f in os.listdir(entry.CSRC) if f.endswith((".cuh", ".h"))] + \
           [os.path.join(entry.ROOT, "include", "tecdsa_b200.h")]
    if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in deps):
        subprocess.check_call(["g++", "-O1", "-w", "-I", HERE, "-I", entry.CSRC, "-shared", "-fPIC", "-o", so, src])
    lib = ctypes.CDLL(so)
    V, I_ = ctypes.c_void_p, ctypes.c_int
    lib.h_commit.argtypes = [V, I_, V, V, I_]
    lib.h_round2.argtypes = [V, I_, V, V, V, V, V, V, V, I_]
    lib.h_validate_pairs.argtypes = [V, I_, V, I_, V, I_, V, I_]
    lib.h_xi.argtypes = [V, I_, V, I_]
    lib.h_dlog_prove.argtypes = [V, V, V, I_]
    lib.h_global_commitments.argtypes = [V, I_, I_, V, I_]
    lib.h_round4.argtypes = [V, I_, I_, V, V, I_]
    lib.h_finish.argtypes = [I_, I_] + [V] * 15 + [I_]
    lib.h_init()
    return lib


class Group:
    """one honest group's Round-3/4 inputs in the kernels' layouts, from the oracle"""

    def __init__(self, t, n, seed):
        rng = random.Random(seed)
        self.t, self.n, self.t1 = t, n, t + 1
        self.u = [rng.randrange(1, Q) for _ in range(n)]
        self.vss = [kg.vss_share(t, n, u, [rng.randrange(1, Q) for _ in range(t)]) for u in self.u]
        self.comm = np.stack([np.stack([pt16(c) for c in v[0].commitments]) for v in self.vss]).astype(np.uint32)   # [n][t1][16]
        self.shares = np.stack([np.stack([L(s, 8) for s in v[1]]) for v in self.vss]).astype(np.uint32)             # [n][n][8]
        self.y = np.ascontiguousarray(self.comm[:, 0, :])
        self.nonce = np.stack([L(rng.randrange(1, Q), 8) for _ in range(n)])

    def pairs(self, hk, y=None):
        ok = np.zeros(self.n * self.n, np.uint8)
        y = self.y if y is None else y
        hk.h_validate_pairs(P(self.comm), self.t1, P(y), 16, P(self.shares), self.n, P(ok), self.n * self.n)
        return ok.reshape(self.n, self.n)

    def round4(self, hk, proof=None):
        x = np.zeros((self.n, 8), np.uint32)
        hk.h_xi(P(self.shares), self.n, P(x), self.n)
        if proof is None:
            proof = np.zeros((self.n, 40), np.uint32)
            hk.h_dlog_prove(P(x), P(self.nonce), P(proof), self.n)
        gcomm = np.zeros((self.t1, 16), np.uint32)
        hk.h_global_commitments(P(self.comm), self.t1, self.n, P(gcomm), 1)
        ok4 = np.zeros(self.n, np.uint8)
        hk.h_round4(P(gcomm), self.t1, self.n, P(proof), P(ok4), self.n)
        return x, proof, gcomm, ok4


@pytest.mark.parametrize("t,n", [(1, 3), (2, 5), (3, 4)])
def test_group_kernels_equal_oracle(hk, t, n):
    g = Group(t, n, 0x4B00 + n)
    assert g.pairs(hk).all()
    x, proof, gcomm, ok4 = g.round4(hk)
    want_x = [sum(v[1][i] for v in g.vss) % Q for i in range(n)]
    assert [I(r) for r in x] == want_x
    glob = [g.vss[0][0].commitments[k] for k in range(t + 1)]
    for v in g.vss[1:]:
        glob = [o.pt_add(a, b) for a, b in zip(glob, v[0].commitments)]
    assert [from16(r) for r in gcomm] == glob
    assert from16(gcomm[0]) == o.pt_mul(G, sum(g.u) % Q)                     # y_sum_s
    assert ok4.all()
    xi = kg.commitments_to_xi([v[0] for v in g.vss])
    assert [from16(proof[i, :16]) for i in range(n)] == xi
    pf = o.dlog_prove(want_x[0], I(g.nonce[0]))
    assert (from16(proof[0, :16]), from16(proof[0, 16:32]), I(proof[0, 32:40])) == (pf.pk, pf.pk_t_rand_commitment, pf.challenge_response)


def _finish(hk, n, t1, st_nt, ok2, pair_ok, ok4, proof=None, gcomm=None):
    E = len(st_nt)
    groups = E // n
    proof = np.arange(E * 40, dtype=np.uint32).reshape(E, 40) + 1 if proof is None else proof
    gcomm = np.arange(groups * t1 * 16, dtype=np.uint32).reshape(groups, t1, 16) + 7 if gcomm is None else gcomm
    o_ = dict(status=np.full(E, 99, np.uint8), bad=np.full(E, 7, np.uint64), complete=np.full(groups, 9, np.uint8), pk=np.ones((E, 16), np.uint32),
              y=np.ones((groups, 16), np.uint32), x=np.ones((E, 8), np.uint32), vss=np.ones((E, t1, 16), np.uint32), n64=np.ones((E, 64), np.uint32),
              st=np.ones((E, 3, 64), np.uint32))
    arrs = [np.ascontiguousarray(a, dtype=np.uint8) for a in (st_nt, ok2, pair_ok, ok4)]
    hk.h_finish(n, t1, *[P(a) for a in arrs], P(proof), P(gcomm), *[P(o_[k]) for k in ("status", "bad", "complete", "pk", "y", "x", "vss", "n64", "st")], E)
    return o_, proof, gcomm


def test_tampering_names_exactly_the_sender(hk):
    t, n = 2, 4
    g = Group(t, n, 0x4B77)
    ones = np.ones(n, np.uint8)
    # a tampered share from sender 2 to receiver 4: receiver 4 alone is INVALID_SS with bit 1
    g.shares[1, 3] = L((I(g.shares[1, 3]) + 1) % Q, 8)
    pair = g.pairs(hk)
    assert pair.sum() == n * n - 1 and not pair[3, 1]
    out, _, _ = _finish(hk, n, t + 1, np.zeros(n), ones, pair.ravel(), ones)
    assert list(out["status"]) == [0, 0, 0, kgg.ST_INVALID_SS] and list(out["bad"]) == [0, 0, 0, 0b10] and out["complete"][0] == 0
    assert not out["x"].any() and not out["pk"].any() and not out["y"].any() and not out["vss"].any()
    # a tampered commitment of sender 3: every receiver fails that sender
    g = Group(t, n, 0x4B77)
    g.comm[2, 2] = pt16(o.pt_mul(G, 5))
    pair = g.pairs(hk)
    assert (pair[:, 2] == 0).all() and pair[:, [0, 1, 3]].all()
    out, _, _ = _finish(hk, n, t + 1, np.zeros(n), ones, pair.ravel(), ones)
    assert list(out["status"]) == [kgg.ST_INVALID_SS] * n and list(out["bad"]) == [0b100] * n
    # a decommitted y that is not commitment 0 (sender 1)
    g = Group(t, n, 0x4B77)
    y = g.y.copy()
    y[0] = pt16(o.pt_mul(G, 3))
    pair = g.pairs(hk, y)
    assert (pair[:, 0] == 0).all() and pair[:, 1:].all()
    # round 4: a pk that is not commitments_to_xi (sender 4), then a DLog proof that does not verify (sender 1)
    g = Group(t, n, 0x4B77)
    x, proof, gcomm, ok4 = g.round4(hk)
    bad_pk = proof.copy()
    other = np.zeros((1, 40), np.uint32)
    hk.h_dlog_prove(P(np.ascontiguousarray(L(12345, 8)[None])), P(np.ascontiguousarray(g.nonce[:1])), P(other), 1)
    bad_pk[3] = other[0]                                                  # a valid proof, for the wrong key
    assert list(g.round4(hk, bad_pk)[3]) == [1, 1, 1, 0]
    bad_pf = proof.copy()
    bad_pf[0, 32] ^= 1
    ok4 = g.round4(hk, bad_pf)[3]
    assert list(ok4) == [0, 1, 1, 1]
    out, _, _ = _finish(hk, n, t + 1, np.zeros(n), ones, np.ones(n * n), ok4, proof=bad_pf, gcomm=gcomm)
    assert list(out["status"]) == [kgg.ST_PROOF] * n and list(out["bad"]) == [1] * n and out["complete"][0] == 0


def test_round2_kernel(hk):
    """the per-sender Round-2 verdict: commitment reopening, proof statuses and the 2047..2048-bit window of N and N~"""
    g = Group(1, 3, 0x4B22)
    blind = np.stack([L(b, 8) for b in (11, 22, 33)])
    com = np.zeros((3, 8), np.uint32)
    hk.h_commit(P(g.comm), 2, P(blind), P(com), 3)
    assert [I(c) for c in com] == [o.hash_commitment(o.bn_from_bytes(o.pt_compress(from16(g.y[i]))), b) for i, b in enumerate((11, 22, 33))]
    n64 = np.stack([L((1 << 2047) + 1, 64), L((1 << 2048) - 1, 64), L((1 << 2045) + 1, 64)])
    nt64 = np.stack([L((1 << 2047) + 3, 64)] * 3)
    ok2 = np.zeros(3, np.uint8)

    def run(st_ck=(0, 0, 0), st_cd=(0,) * 6, com_=com, n_=n64):
        hk.h_round2(P(g.y), 16, P(blind), P(com_), P(np.array(st_ck, np.uint8)), P(n_), P(nt64), P(np.array(st_cd, np.uint8)), P(ok2), 3)
        return list(ok2)

    assert run() == [1, 1, 0]                                              # party 3: a 2046-bit N
    assert run(st_ck=(10, 0, 0)) == [0, 1, 0]
    assert run(st_cd=(0, 0, 0, 0, 10, 0)) == [1, 0, 0]                     # second proof of party 2
    bad_com = com.copy(); bad_com[0, 0] ^= 1
    assert run(com_=bad_com) == [0, 1, 0]


def test_status_precedence(hk):
    """the first failing round decides, per group; the other group of the batch is untouched"""
    n, t1 = 3, 2
    ok = np.ones(2 * n, np.uint8)
    pair = np.ones(2 * n * n, np.uint8)
    # group 0: an uninvertible xhi at party 2 AND a failing broadcast of party 1 AND a failing pair AND a failing DLog proof
    st_nt = np.array([0, 4, 0, 0, 0, 0]); ok2 = ok.copy(); ok2[0] = 0; pr = pair.copy(); pr[2 * n + 1] = 0; ok4 = ok.copy(); ok4[2] = 0
    out, proof, gcomm = _finish(hk, n, t1, st_nt, ok2, pr, ok4)
    assert list(out["status"]) == [0, kgg.ST_NOT_INVERTIBLE, 0, 0, 0, 0] and list(out["bad"]) == [0] * 6 and list(out["complete"]) == [0, 1]
    assert not out["pk"][:3].any() and (out["pk"][3:] == proof[3:, :16]).all() and (out["y"][1] == gcomm[1, 0]).all() and not out["y"][0].any()
    assert (out["x"][3:] == 1).all() and not out["x"][:3].any()
    st_nt[1] = 0
    out, _, _ = _finish(hk, n, t1, st_nt, ok2, pr, ok4)
    assert list(out["status"][:3]) == [kgg.ST_INVALID_KEY] * 3 and list(out["bad"][:3]) == [1] * 3
    ok2[0] = 1
    out, _, _ = _finish(hk, n, t1, st_nt, ok2, pr, ok4)
    assert list(out["status"][:3]) == [0, 0, kgg.ST_INVALID_SS] and list(out["bad"][:3]) == [0, 0, 0b10]
    pr[2 * n + 1] = 1
    out, _, _ = _finish(hk, n, t1, st_nt, ok2, pr, ok4)
    assert list(out["status"][:3]) == [kgg.ST_PROOF] * 3 and list(out["bad"][:3]) == [0b100] * 3
    assert list(out["complete"]) == [0, 1] and list(out["status"][3:]) == [0, 0, 0]


# ------------------------------------------------------------------------------------------------ ABI
def test_keygen_export_everywhere(pkg):
    hdr = open(os.path.join(entry.ROOT, "include", "tecdsa_b200.h")).read()
    assert re.search(r"int tecdsa_gg20_keygen_batch\(tecdsa_ctx\* ctx, int t, int n, size_t groups, int mem, const tecdsa_keygen_in\* in,", hdr)
    assert "tecdsa_gg20_keygen_batch" in pkg.EXPORTS
    ffi = open(os.path.join(entry.ROOT, "bindings", "rust", "src", "ffi.rs")).read()
    assert "pub fn tecdsa_gg20_keygen_batch(ctx: *mut tecdsa_ctx, t: c_int, n: c_int, groups: usize, mem: c_int, in_: *const tecdsa_keygen_in," in ffi
    assert "pub struct tecdsa_keygen_in {" in ffi and "pub bad_actors: *mut u64," in ffi
    # the stream ids of the keygen inputs are disjoint from the offline record's (0..32)
    ids = [int(v) for v in re.findall(r"TECDSA_RNDS_KG_\w+ = (\d+)", hdr)]
    assert len(ids) == 7 and min(ids) > 32 and len(set(ids)) == 7


def test_rust_ffi_is_the_generated_file(tmp_path, monkeypatch):
    """bindings/rust/src/ffi.rs is exactly what tools/gen_rust_ffi.py writes from the header: every declaration and every struct's
    fields, so a header change without regeneration fails here"""
    import importlib.util
    spec = importlib.util.spec_from_file_location("gen_rust_ffi", os.path.join(entry.ROOT, "tools", "gen_rust_ffi.py"))
    gen_ffi = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen_ffi)
    monkeypatch.setattr(gen_ffi, "OUT", str(tmp_path / "ffi.rs"))
    gen_ffi.main()
    assert (tmp_path / "ffi.rs").read_text() == open(os.path.join(entry.ROOT, "bindings", "rust", "src", "ffi.rs")).read()
