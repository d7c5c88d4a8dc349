"""GPU: the seeded sampler through the C ABI against oracle/seeded_sampling.py — tecdsa_sample_batch for every kind, the whole
randomness record of tecdsa_gg20_sample_randomness, sharding invariance, the sampled record through the offline stage and the
online step (host buffers and the device-resident chain), and gg20_general.sample_rnd through the size-generic driver."""
import ctypes
import math
import random

import numpy as np
import pytest

from oracle import gg20_general_oracle as gen
from oracle import gg20_oracle as o
from oracle import seeded_sampling as ss
from tests import test_gg20_general as tg
from tests.golden import fixtures

pytestmark = pytest.mark.gpu
SEED = bytes(range(7, 39))
Q = o.Q
KIND = {0: "bits", 1: "below", 2: "unit", 3: "range1", 4: "scalar"}


def _raw_sample(eng, pkg, seed, first_id, stream, kind, bits, bound, idx, n_bound, limbs, out, status, count, mem):
    eng.sample(pkg.SAMPLE_SCALAR, 1, SEED)                      # binds the argument types
    sw = None if seed is None else pkg.seed_words(seed)
    return eng.lib.tecdsa_sample_batch(eng._ctx, pkg._ptr(sw), first_id, stream, kind, bits, pkg._ptr(bound), pkg._ptr(idx), n_bound, limbs, pkg._ptr(out),
                                       pkg._ptr(status), count, mem)


def test_sample_batch_every_kind_equals_oracle(engine, pkg):
    import torch
    rng = random.Random(0x5A)
    moduli = [lk.dk.p * lk.dk.q for ks in fixtures.load_edge_keysets() + fixtures.load_all_keysets()[:1] for lk in ks]
    n = 1024
    # per-element bounds
    for kind, count, bounds in ((pkg.SAMPLE_BELOW, n, [rng.choice(moduli) >> rng.choice([0, 0, 1, 33, 700]) for _ in range(n)]),
                                (pkg.SAMPLE_RANGE1, n, [rng.choice(moduli) for _ in range(n)]),
                                (pkg.SAMPLE_UNIT, 256, [rng.choice(moduli + [3 * 5 * 7 * 11 * 13 * 2 ** 2000]) for _ in range(256)])):
        got, st = engine.sample(kind, count, SEED, stream=50 + kind, first_id=2 ** 33, bound=bounds, limbs=64)
        want = [ss.sample(SEED, 50 + kind, 2 ** 33 + i, KIND[kind], bounds[i]) for i in range(count)]
        assert not st.any() and got == [w[0] for w in want]
        assert kind != pkg.SAMPLE_UNIT or all(math.gcd(v, b) == 1 for v, b in zip(got, bounds))
    # a shared table through bound_idx, TECDSA_DEVICE buffers, 88-limb bounds (q^3 N~)
    table = [Q ** 3 * lk.h1_h2_n_tilde_vec[lk.i - 1].N for lk in fixtures.load_keyset(0)]
    idx = [rng.randrange(3) for _ in range(n)]
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.int32)).cuda()
    out, st = torch.zeros((n, 88), dtype=torch.int32, device="cuda"), torch.full((n,), 255, dtype=torch.uint8, device="cuda")
    assert _raw_sample(engine, pkg, SEED, 5, 9, pkg.SAMPLE_BELOW, 0, T(pkg.ints_to_limbs(table, 88)), T(np.asarray(idx, np.uint32)), 3, 88, out, st, n, pkg.DEVICE) == 0
    engine.sync()
    assert not st.cpu().numpy().any()
    assert pkg.limbs_to_ints(out.cpu().numpy().view(np.uint32)) == [ss.sample(SEED, 9, 5 + i, "below", table[idx[i]])[0] for i in range(n)]
    got, st = engine.sample(pkg.SAMPLE_BELOW, n, SEED, stream=9, first_id=5, bound=table, bound_idx=idx, limbs=88)
    assert not st.any() and got == pkg.limbs_to_ints(out.cpu().numpy().view(np.uint32))
    got, st = engine.sample(pkg.SAMPLE_SCALAR, 2 * n, SEED, stream=1, first_id=0)
    assert not st.any() and got == [ss.sample(SEED, 1, i, "scalar")[0] for i in range(2 * n)]
    for bits, limbs in ((256, 8), (1, 4), (2047, 64), (4096, 128)):
        got, st = engine.sample(pkg.SAMPLE_BITS, 64, SEED, stream=2, first_id=bits, bits=bits, limbs=limbs)
        assert not st.any() and got == [ss.sample(SEED, 2, bits + i, "bits", bits=bits)[0] for i in range(64)]
    # degenerate bounds: that element gets the status and a zero value, its neighbours their values
    for kind, bad in ((pkg.SAMPLE_BELOW, [0]), (pkg.SAMPLE_UNIT, [0, 1]), (pkg.SAMPLE_RANGE1, [0, 1, 2])):
        bounds = [moduli[0]] + bad + [moduli[1]]
        got, st = engine.sample(kind, len(bounds), SEED, stream=3, bound=bounds, limbs=64)
        assert list(st) == [0] + [pkg.ST_SAMPLING] * len(bad) + [0] and got[1:-1] == [0] * len(bad)
        assert got[0] == ss.sample(SEED, 3, 0, KIND[kind], moduli[0])[0] and got[-1] == ss.sample(SEED, 3, len(bounds) - 1, KIND[kind], moduli[1])[0]
    got, st = engine.sample(pkg.SAMPLE_BELOW, 3, SEED, bound=table, bound_idx=[0, 3, 2], limbs=88)       # an index outside the table
    assert list(st) == [0, pkg.ST_SAMPLING, 0] and got[1] == 0
    # argument errors, before anything is touched
    o8, s8, b8 = np.full((4, 8), 7, np.uint32), np.full(4, 255, np.uint8), pkg.ints_to_limbs([5] * 4, 8)
    E = -1
    assert _raw_sample(engine, pkg, SEED, 0, 0, 5, 0, b8, None, 0, 8, o8, s8, 4, pkg.HOST) == E
    assert _raw_sample(engine, pkg, SEED, 0, 0, -1, 0, b8, None, 0, 8, o8, s8, 4, pkg.HOST) == E
    assert _raw_sample(engine, pkg, SEED, 0, 0, pkg.SAMPLE_BELOW, 0, b8, None, 0, 8, o8, s8, 4, 2) == E
    assert _raw_sample(engine, pkg, None, 0, 0, pkg.SAMPLE_BELOW, 0, b8, None, 0, 8, o8, s8, 4, pkg.HOST) == E
    assert _raw_sample(engine, pkg, SEED, 0, 0, pkg.SAMPLE_BELOW, 0, None, None, 0, 8, o8, s8, 4, pkg.HOST) == E
    assert _raw_sample(engine, pkg, SEED, 0, 0, pkg.SAMPLE_BELOW, 0, b8, None, 0, 8, None, s8, 4, pkg.HOST) == E
    assert _raw_sample(engine, pkg, SEED, 0, 0, pkg.SAMPLE_BELOW, 0, b8, None, 0, 8, o8, None, 4, pkg.HOST) == E
    assert _raw_sample(engine, pkg, SEED, 0, 0, pkg.SAMPLE_BELOW, 0, b8, None, 0, 129, o8, s8, 4, pkg.HOST) == E
    assert _raw_sample(engine, pkg, SEED, 0, 0, pkg.SAMPLE_BITS, 257, None, None, 0, 8, o8, s8, 4, pkg.HOST) == E
    assert _raw_sample(engine, pkg, SEED, 0, 0, pkg.SAMPLE_BITS, 0, None, None, 0, 8, o8, s8, 4, pkg.HOST) == E
    assert _raw_sample(engine, pkg, SEED, 0, 0, pkg.SAMPLE_SCALAR, 0, None, None, 0, 4, o8, s8, 4, pkg.HOST) == E
    assert (o8 == 7).all() and (s8 == 255).all()


def _sessions(rng, n_keysets, n):
    pairs = [(0, 1), (0, 2), (1, 2), (1, 0), (2, 0), (2, 1)]
    return np.array([(rng.randrange(n_keysets), *rng.choice(pairs)) for _ in range(n)], dtype=np.uint32)


def _oracle_record(pkg, keysets, sessions, first_unit):
    from mpecdsa_b200 import gg20
    units = []
    for s, (k, a, b) in enumerate(sessions.tolist()):
        keys, s_l = [keysets[k][a], keysets[k][b]], [a + 1, b + 1]
        units += [ss.sample_unit_seeded(SEED, first_unit + 2 * s + p, keys, s_l, p) for p in range(2)]
    return units, gg20.pack_randomness(units)


@pytest.fixture(scope="module")
def mixed(engine):
    from mpecdsa_b200 import gg20
    keysets = fixtures.load_all_keysets()[:3] + fixtures.load_edge_keysets()
    ks = gg20.KeySets(engine, keysets)
    yield keysets, ks
    ks.free()


def test_gg20_record_equals_oracle_and_sharding_is_invariant(engine, pkg, mixed):
    from mpecdsa_b200 import gg20
    keysets, ks = mixed
    n, first = 256, 2 ** 32 - 100                       # unit ids cross the 32-bit boundary of the element id
    sessions = _sessions(random.Random(1), len(keysets), n)
    rnd, st = gg20.sample_randomness(engine, ks, sessions, seed=SEED, first_unit=first)
    assert not st.any()
    _, want = _oracle_record(pkg, keysets, sessions, first)
    assert np.array_equal(rnd, want)
    # one call over U units == two calls over the halves with first_unit shifted by the units before them
    lo, _ = gg20.sample_randomness(engine, ks, sessions[:n // 2], seed=SEED, first_unit=first)
    hi, _ = gg20.sample_randomness(engine, ks, sessions[n // 2:], seed=SEED, first_unit=first + n)
    assert np.array_equal(np.concatenate([lo, hi]), rnd)
    other, _ = gg20.sample_randomness(engine, ks, sessions[:4])                  # seed=None: fresh, never the caller's
    assert not np.array_equal(other[:, :16], rnd[:8, :16])
    # a descriptor that names no key row or the same party twice: status and a zero record for both units, neighbours untouched
    bad = sessions[:4].copy(); bad[1] = (len(keysets), 0, 1); bad[2] = (0, 1, 1)
    r2, s2 = gg20.sample_randomness(engine, ks, bad, seed=SEED, first_unit=first)
    assert list(s2) == [0, 0] + [pkg.ST_SAMPLING] * 4 + [0, 0] and not r2[2:6].any()
    assert np.array_equal(r2[:2], rnd[:2]) and np.array_equal(r2[6:8], rnd[6:8])
    for args in ((None, sessions, SEED), (ks.handle, None, SEED), (ks.handle, sessions, None)):
        sw = None if args[2] is None else pkg.seed_words(args[2])
        assert engine.lib.tecdsa_gg20_sample_randomness(engine._ctx, args[0], pkg._ptr(args[1]), 4, pkg._ptr(sw), 0, pkg._ptr(r2), pkg._ptr(s2), pkg.HOST) == -1
    assert engine.lib.tecdsa_gg20_sample_randomness(engine._ctx, ks.handle, pkg._ptr(sessions), 4, pkg._ptr(pkg.seed_words(SEED)), 0, pkg._ptr(r2), pkg._ptr(s2), 7) == -1


def _be(limbs):
    return np.ascontiguousarray(limbs[:, ::-1]).astype(">u4").view(np.uint8).reshape(limbs.shape[0], 32)


def test_sampled_record_through_the_offline_stage_and_the_online_step(engine, pkg, mixed):
    import torch
    from cryptography.hazmat.primitives import hashes
    from cryptography.hazmat.primitives.asymmetric import ec, utils
    from mpecdsa_b200 import gg20
    from oracle import twin
    keysets, ks = mixed
    n = 24
    sessions = _sessions(random.Random(2), len(keysets), n)
    assert {3, 4, 5} <= set(sessions[:, 0].tolist())                              # edge keys take part
    rnd, st = gg20.sample_randomness(engine, ks, sessions, seed=SEED)
    units, want_rnd = _oracle_record(pkg, keysets, sessions, 0)
    assert not st.any() and np.array_equal(rnd, want_rnd)
    res = gg20.offline_batch(engine, ks, sessions, rnd)
    assert not res.status.any()
    want = twin.offline_batch(twin.KeyTables(keysets), sessions, want_rnd, 8)
    assert not want.status.any() and np.array_equal(res.digest, want.digest) and np.array_equal(res.R, want.R) and np.array_equal(res.sigma, want.sigma)
    for s in (0, n - 1):                                                          # and the Python restatement on the oracle's own values
        k, a, b = sessions[s].tolist()
        ref = o.offline_session([keysets[k][a], keysets[k][b]], [a + 1, b + 1], units[2 * s:2 * s + 2])
        for p in range(2):
            assert int.from_bytes(res.digest[2 * s + p].tobytes(), "little").to_bytes(32, "big") == ref[p].transcript
    # the device-resident chain: sample -> offline -> pack records, the record of randomness never in host memory
    U = 2 * n
    Z = lambda *shape, dt=torch.int32: torch.zeros(shape, dtype=dt, device="cuda")
    d_sess = torch.from_numpy(sessions.view(np.int32)).cuda()
    d_rnd, d_sst, d_st, d_R, d_sig, d_t, d_dig = Z(U, gg20.RND_LIMBS), Z(U, dt=torch.uint8), Z(U, dt=torch.uint8), Z(U, 16), Z(U, 8), Z(U, 32), Z(U, 8)
    d_rec = Z(U, pkg.REC_BYTES, dt=torch.uint8)
    gg20.sample_randomness(engine, ks, d_sess, seed=SEED, mem=pkg.DEVICE, rnd=d_rnd, status=d_sst)
    gg20.offline_raw(engine, ks, d_sess, n, d_rnd, d_st, d_R, d_sig, d_t, d_dig, mem=pkg.DEVICE)
    engine.pack_records(d_st, d_R, d_sig, d_t, d_dig, d_rnd, U, d_rec)
    engine.sync()
    rec = d_rec.cpu().numpy()
    assert not d_sst.cpu().numpy().any() and not rec[:, 0].any()
    assert np.array_equal(rec[:, 164:196], _be(want.digest)) and np.array_equal(rec[:, 66:98], _be(want.k))
    k_limbs = np.ascontiguousarray(rec[:, 66:98].reshape(U, 8, 4)[:, ::-1, ::-1]).view("<u4").reshape(U, 8)
    m = o.sha256_bigints([o.bn_from_bytes(b"seeded")])
    msg = np.tile(np.frombuffer(m.to_bytes(32, "little"), dtype="<u4"), (n, 1))
    sig = gg20.sign_batch(engine, ks, sessions, msg, d_R.cpu().numpy().view(np.uint32), d_sig.cpu().numpy().view(np.uint32), k_limbs)
    assert not sig["status"].any()
    for s in range(n):
        r_, s_ = pkg.limbs_to_ints(sig["r"][s:s + 1])[0], pkg.limbs_to_ints(sig["s"][s:s + 1])[0]
        y = keysets[int(sessions[s, 0])][0].y_sum_s
        pub = ec.EllipticCurvePublicNumbers(y[0], y[1], ec.SECP256K1()).public_key()
        pub.verify(utils.encode_dss_signature(r_, s_), m.to_bytes(32, "big"), ec.ECDSA(utils.Prehashed(hashes.SHA256())))


def _party_randomness(rnd, u, ttag):
    P1 = ttag - 1
    r = gen.PartyRandomness(gamma_i=rnd["gamma"][u], k_i=rnd["k"][u], blind=rnd["blind"][u], r_k=rnd["r_k"][u], alice=list(rnd["alice"][u]),
                            l=rnd["l"][u], ped_s1=rnd["ped_s1"][u], ped_s2=rnd["ped_s2"][u], heg_s1=rnd["heg_s1"][u], heg_s2=rnd["heg_s2"][u])
    for f in ("beta_tag_gamma", "r_gamma", "nonce_gamma_b", "nonce_gamma_beta", "beta_tag_w", "r_w", "nonce_w_b", "nonce_w_beta", "pdl"):
        setattr(r, f, [rnd[f][u * P1 + j] for j in range(P1)])
    return r


def test_sample_rnd_through_the_general_driver(engine, pkg):
    from mpecdsa_b200 import gg20, gg20_general
    keysets = fixtures.load_all_keysets()[:2]
    ks = gg20.KeySets(engine, keysets)
    rng = random.Random(0x5EED)
    key5 = tg._five_party_key(keysets, rng)
    cases = [([keysets[1][i - 1] for i in (3, 1, 2)], [3, 1, 2], lambda lk, j: 3 + j), ([key5[i - 1] for i in (5, 2, 3)], [5, 2, 3], lambda lk, j: j)]
    try:
        for keys, s_l, row_of in cases:
            ttag, l_s = len(s_l), [i - 1 for i in s_l]
            key_rows, all_rows = [row_of(lk, lk.i - 1) for lk in keys], [[row_of(lk, j) for j in range(lk.n)] for lk in keys]
            lam = [o.lagrange_at_zero(l_s[p], l_s) for p in range(ttag)]
            w, g_w, y = [lam[p] * lk.x_i % Q for p, lk in enumerate(keys)], [o.pt_mul(lk.pk_vec[l_s[p]], lam[p]) for p, lk in enumerate(keys)], [lk.y_sum_s for lk in keys]
            rnd = gg20_general.sample_rnd(engine, ks, ttag, key_rows, all_rows, seed=SEED)
            out = gg20_general.offline_batch(engine, ks, ttag, key_rows, all_rows, w, g_w, y, rnd)
            want = gen.offline_session(keys, s_l, [_party_randomness(rnd, p, ttag) for p in range(ttag)])
            assert tg._signature_ok(want, keys[0].y_sum_s, rng)
            for p, wv in enumerate(want):
                assert int(out["status"][p]) == wv.status == 0
                assert (out["R"][p], out["sigma"][p], out["k"][p], out["T"][p]) == (wv.R, wv.sigma_i, wv.k_i, wv.t_vec[p])
    finally:
        ks.free()
