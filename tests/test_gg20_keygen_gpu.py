"""GG20 key generation as one device call (tecdsa_gg20_keygen_batch) on the GPU: every output equal to the party-by-party group
oracle (tests/keygen_group.py) for several (t, n) and several groups per call, the failure paths and their isolation from the other
groups of a batch, the keys through signing and the wire format, TECDSA_DEVICE buffers byte-identical to TECDSA_HOST (with the inputs
sampled on the device), and the seeded sampling of the inputs against oracle/seeded_sampling.py."""
import functools
import random

import numpy as np
import pytest

from oracle import gg20_oracle as o
from oracle import keygen_oracle as kg
from oracle import seeded_sampling as ss
from tests import keygen_group as kgg
from tests.golden import fixtures

pytestmark = pytest.mark.gpu
Q = o.Q
SEED = bytes(range(7, 39))


@functools.lru_cache(maxsize=None)
def _prime_pair(seed):
    return kgg.prime_pair(seed)


def _rows():
    return [lk for ks in fixtures.load_all_keysets() for lk in ks]


def _primes(n, groups, shift=0, edge=False):
    """Paillier primes from the fixture rows (keys_edge.json rows for group 1 when edge: 2047-bit N, unbalanced factors); N~ primes
    made on the CPU for group 0 and taken from other fixture rows for the rest"""
    rows, erows = _rows(), [lk for ks in fixtures.load_edge_keysets() for lk in ks]
    out = []
    for g in range(groups):
        for i in range(n):
            src = erows[i % len(erows)] if edge and g == 1 else rows[(shift + g * n + i) % 12]
            nt = _prime_pair(1000 + shift + i) if g == 0 else (rows[12 + (shift + g * n + i) % 12].dk.p, rows[12 + (shift + g * n + i) % 12].dk.q)
            out.append(((src.dk.p, src.dk.q), nt))
    return out


def _inputs(t, n, primes, seed):
    rng = random.Random(seed)
    return [kgg.random_inputs(t, pr[1], rng) for pr in primes]


def _run(engine, t, n, primes, rnd, mem=0):
    from mpecdsa_b200 import keygen
    return keygen.keygen_batch(engine, t, n, [p[0] for p in primes], [p[1] for p in primes], keygen.pack_randomness(t, rnd), mem=mem)


def _check_group(res, t, n, g, want_keys, want_status, want_bad):
    rows = range(g * n, g * n + n)
    assert [int(res.status[r]) for r in rows] == want_status
    assert [int(res.bad_actors[r]) for r in rows] == want_bad
    assert int(res.complete[g]) == (1 if want_keys[0] is not None else 0)
    for i, r in enumerate(rows):
        got, want = res.keys[r], want_keys[i]
        if want is None:
            assert got is None
            assert not res.out["x_i"][r].any() and not res.out["vss"][r].any() and not res.out["n"][r].any() and not res.out["dlog_st"][r].any()
            assert not res.out["pk"][g].any() and not res.out["y"][g].any()
            continue
        assert (got.i, got.t, got.n, got.x_i, got.dk.p, got.dk.q) == (want.i, want.t, want.n, want.x_i, want.dk.p, want.dk.q)
        assert got.pk_vec == want.pk_vec and got.y_sum_s == want.y_sum_s and got.vss_commitments == want.vss_commitments
        assert [e.n for e in got.paillier_key_vec] == [e.n for e in want.paillier_key_vec]
        assert [(s.N, s.g, s.ni) for s in got.h1_h2_n_tilde_vec] == [(s.N, s.g, s.ni) for s in want.h1_h2_n_tilde_vec]


@pytest.mark.parametrize("t,n", [(1, 3), (2, 5), (3, 4), (1, 2)])
def test_keygen_parity(engine, t, n):
    groups = 2
    primes = _primes(n, groups, shift=n, edge=(t, n) == (1, 3))
    rnd = _inputs(t, n, primes, 0x7000 + 16 * t + n)
    res = _run(engine, t, n, primes, rnd)
    assert list(res.complete) == [1] * groups
    for g in range(groups):
        keys, status, bad = kgg.keygen_group(t, n, primes[g * n:(g + 1) * n], rnd[g * n:(g + 1) * n])
        _check_group(res, t, n, g, keys, status, bad)


def test_keygen_failure_paths_are_isolated(engine, pkg):
    t, n = 1, 3
    primes = _primes(n, 3)
    rnd = _inputs(t, n, primes, 0x7100)
    clean = _run(engine, t, n, primes[:3] + primes[6:], rnd[:3] + rnd[6:])
    cases = []
    p = list(primes)
    p[4] = ((p[4][0][0] >> 2 | 1, p[4][0][1]), p[4][1])                 # party 2 of group 1: a 2046-bit N
    cases.append((p, rnd, [pkg.ST_INVALID_KEY] * 3, [0b010] * 3))
    p = list(primes)
    p[5] = ((p[5][0][0], p[5][0][0]), p[5][1])                         # party 3 of group 1: p = q
    cases.append((p, rnd, [pkg.ST_INVALID_KEY] * 3, [0b100] * 3))
    r = [dict(x) for x in rnd]
    r[3]["xhi"] = 2 * (r[3]["xhi"] // 2)                                # party 1 of group 1: an even xhi has no inverse mod phi
    cases.append((primes, r, [pkg.ST_NOT_INVERTIBLE, 0, 0], [0, 0, 0]))
    for p, r, st, bad in cases:
        res = _run(engine, t, n, p, r)
        assert list(res.complete) == [1, 0, 1]
        want = kgg.keygen_group(t, n, p[3:6], r[3:6])
        assert want[1:] == (st, bad)
        _check_group(res, t, n, 1, want[0], st, bad)
        for f, a in res.out.items():
            b = clean.out[f]
            per = a.shape[0] // 3
            assert np.array_equal(np.concatenate([a[:per], a[2 * per:]]), b), f


def test_keygen_to_signatures(engine, pkg):
    """(1, 3) keys through gg20.KeySets, the seeded offline stage and the online step; (2, 5) keys through gg20_general with three
    signers; every signature verifies under OpenSSL against y_sum_s; every key round-trips through the wire format"""
    from cryptography.hazmat.primitives import hashes
    from cryptography.hazmat.primitives.asymmetric import ec, utils
    from mpecdsa_b200 import gg20, gg20_general, wire
    from tests import test_gg20_general as tg

    def openssl_ok(y, r_, s_, m):
        pub = ec.EllipticCurvePublicNumbers(y[0], y[1], ec.SECP256K1()).public_key()
        pub.verify(utils.encode_dss_signature(r_, s_), m.to_bytes(32, "big"), ec.ECDSA(utils.Prehashed(hashes.SHA256())))

    primes = _primes(3, 2)
    res = _run(engine, 1, 3, primes, _inputs(1, 3, primes, 0x7200))
    assert list(res.complete) == [1, 1]
    keysets = [res.keys[0:3], res.keys[3:6]]
    ks = gg20.KeySets(engine, keysets)
    sessions = np.array([[0, 0, 2], [1, 1, 0]], dtype=np.uint32)
    rnd, st = gg20.sample_randomness(engine, ks, sessions, seed=SEED)
    assert not st.any()
    off = gg20.offline_batch(engine, ks, sessions, rnd)
    assert not off.status.any()
    msg = [random.Random(s).getrandbits(256) % Q for s in range(2)]
    msg_l = pkg.ints_to_limbs(msg, 8)
    sig = gg20.sign_batch(engine, ks, sessions, msg_l, off.R, off.sigma, np.ascontiguousarray(rnd[:, 8:16]))      # k_i = TECDSA_RND_K
    assert not sig["status"].any()
    for s, (r_, s_) in enumerate(zip(pkg.limbs_to_ints(sig["r"]), pkg.limbs_to_ints(sig["s"]))):
        openssl_ok(keysets[s][0].y_sum_s, r_, s_, msg[s])
    ks.free()
    # (2, 5): signers 5, 2, 3 through the size-generic driver
    primes = _primes(5, 1)
    res5 = _run(engine, 2, 5, primes, _inputs(2, 5, primes, 0x7205))
    key5 = res5.keys
    ks5 = gg20.KeySets(engine, [key5[0:3], key5[3:5] + key5[0:1]])
    rng = random.Random(0x7206)
    s_l = [5, 2, 3]
    keys = [key5[i - 1] for i in s_l]
    srnd = [tg._party_randomness(rng, lk, [s_l[gen_ind(p, j)] - 1 for j in range(2)]) for p, lk in enumerate(keys)]
    out = gg20_general.offline_batch(engine, ks5, *tg._flatten([(keys, s_l, srnd)], lambda lk, j: j))
    assert list(out["status"]) == [0, 0, 0]
    m = rng.getrandbits(256) % Q
    r_, s_, _ = o.output_signature(out["R"][0], [o.local_sig(out["k"][p], m, out["R"][p], out["sigma"][p]) for p in range(3)])
    openssl_ok(key5[0].y_sum_s, r_, s_, m)
    ks5.free()
    for lk in res.keys + key5:
        doc = wire.local_key(lk, lk.vss_commitments)
        back = wire.load_local_key(doc, lambda b: engine.point_decompress([b])[0])
        assert back == lk


def gen_ind(p, j):
    from oracle import gg20_general_oracle as gen
    return gen._ind(p, j)


def test_keygen_device_buffers_equal_host(engine, pkg):
    import torch
    from mpecdsa_b200 import keygen
    t, n = 2, 4
    primes = _primes(n, 2)
    nt = [p[1] for p in primes]
    rec_h = keygen.sample_randomness(engine, t, n, nt, SEED, first_id=5)
    rec_d = keygen.sample_randomness(engine, t, n, nt, SEED, first_id=5, mem=pkg.DEVICE)
    for f in rec_h:
        assert isinstance(rec_d[f], torch.Tensor) and rec_d[f].is_cuda
        assert np.array_equal(rec_h[f], keygen._host(rec_d[f])), f
    res_h = keygen.keygen_batch(engine, t, n, [p[0] for p in primes], nt, rec_h)
    res_d = keygen.keygen_batch(engine, t, n, [p[0] for p in primes], nt, rec_d, mem=pkg.DEVICE)
    assert list(res_h.complete) == [1, 1] and res_d.keys is None
    for f, a in res_h.out.items():
        assert res_d.out[f].is_cuda and np.array_equal(a, keygen._host(res_d.out[f])), f
    # the device-sampled record reproduces the oracle end to end
    rnd = [{"u": int(keygen.limbs_to_ints(rec_h["u"][e:e + 1])[0]), "coeffs": keygen.limbs_to_ints(rec_h["coeffs"][e]),
            "blind": keygen.limbs_to_ints(rec_h["blind"][e:e + 1])[0], "h1": keygen.limbs_to_ints(rec_h["h1"][e:e + 1])[0],
            "xhi": keygen.limbs_to_ints(rec_h["xhi"][e:e + 1])[0], "cdl_nonce": tuple(keygen.limbs_to_ints(rec_h["cdl_nonce"][e])),
            "dlog_nonce": keygen.limbs_to_ints(rec_h["dlog_nonce"][e:e + 1])[0]} for e in range(2 * n)]
    keys, status, bad = kgg.keygen_group(t, n, primes[:n], rnd[:n])
    _check_group(res_h, t, n, 0, keys, status, bad)


def test_keygen_sampling(engine):
    from mpecdsa_b200 import keygen
    t, n = 2, 3
    primes = _primes(n, 2)
    nt = [p[1] for p in primes]
    a = keygen.sample_randomness(engine, t, n, nt, SEED)
    b = keygen.sample_randomness(engine, t, n, nt, SEED)
    assert all(np.array_equal(a[f], b[f]) for f in a)
    # split by first_id: the second half of the batch drawn on its own
    half = keygen.sample_randomness(engine, t, n, nt[n:], SEED, first_id=n)
    assert all(np.array_equal(a[f][n:], half[f]) for f in a)
    other = keygen.sample_randomness(engine, t, n, nt, bytes(32))
    assert not np.array_equal(a["u"], other["u"])
    I = lambda row: int.from_bytes(np.ascontiguousarray(row).tobytes(), "little")
    for e in (0, 4):
        pt, qt = nt[e]
        want = {"u": ss.sample(SEED, keygen.RNDS_KG_U, e, "scalar"), "blind": ss.sample(SEED, keygen.RNDS_KG_BLIND, e, "bits", bits=256),
                "h1": ss.sample(SEED, keygen.RNDS_KG_H1, e, "below", bound=pt * qt),
                "xhi": ss.sample(SEED, keygen.RNDS_KG_XHI, e, "unit", bound=(pt - 1) * (qt - 1)),
                "dlog_nonce": ss.sample(SEED, keygen.RNDS_KG_DLOG, e, "scalar")}
        for f, (v, ok, _) in want.items():
            assert ok and I(a[f][e]) == v, f
        for k in range(t):
            assert I(a["coeffs"][e, k]) == ss.sample(SEED, keygen.RNDS_KG_COEFF, (k << 32) + e, "scalar")[0]
        for k in range(2):
            assert I(a["cdl_nonce"][e, k]) == ss.sample(SEED, keygen.RNDS_KG_CDL, (k << 32) + e, "bits", bits=512)[0]
    assert all(kgg.gcd(I(a["xhi"][e]), (nt[e][0] - 1) * (nt[e][1] - 1)) == 1 for e in range(2 * n))
