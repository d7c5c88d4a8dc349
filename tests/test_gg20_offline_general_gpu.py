"""GPU tests of the GG20 offline stage for any signing set as one call (tecdsa_gg20_offline_general_batch): parity with the
size-generic oracle for (t, n, s_l) from two of two to five of eight, several sessions and key sets per call over the fixture and
keys_edge.json Paillier / N~ material; equality with the Python driver (gg20_general.offline_batch) on 64 sessions and with the fused
two-signer call; the failure paths; DEVICE against HOST buffers; the sampled inputs against sample_rnd; the executed work against
the Python driver; key sets of any size; and keys from tecdsa_gg20_keygen_batch through to signatures OpenSSL accepts."""
import random

import numpy as np
import pytest

from oracle import gg20_general_oracle as gen
from oracle import gg20_oracle as o
from tests.golden import fixtures

Q, G = o.Q, o.G
SEED = bytes(range(32))
pytestmark = pytest.mark.gpu


def _key(rows, t, n, rng):
    """a (t, n) key over the Paillier keys / N~ setups of `rows` (n LocalKeys of the fixtures): fresh degree-t Shamir sharing"""
    coef = [rng.randrange(1, Q) for _ in range(t + 1)]
    x = [sum(c * pow(i + 1, k, Q) for k, c in enumerate(coef)) % Q for i in range(n)]
    eks = [o.EncryptionKey(lk.dk.p * lk.dk.q, (lk.dk.p * lk.dk.q) ** 2) for lk in rows]
    sts = [lk.h1_h2_n_tilde_vec[lk.i - 1] for lk in rows]
    pks = [o.pt_mul(G, xi) for xi in x]
    return [o.LocalKey(i=i + 1, t=t, n=n, x_i=x[i], dk=rows[i].dk, pk_vec=pks, paillier_key_vec=eks, h1_h2_n_tilde_vec=sts, y_sum_s=o.pt_mul(G, coef[0]))
            for i in range(n)]


def _rows(edge=False):
    return [lk for ks in (fixtures.load_edge_keysets() if edge else fixtures.load_all_keysets()) for lk in ks]


def _host(a):
    from mpecdsa_b200.keygen import _host as h
    return h(a)


def _party(inp, u, T, P):
    I = lambda f, *ix: int.from_bytes(np.ascontiguousarray(_host(inp[f])[ix]).tobytes(), "little")
    r = gen.PartyRandomness(gamma_i=I("gamma", u), k_i=I("k", u), blind=I("blind", u), r_k=I("r_k", u), l=I("l", u), ped_s1=I("ped_s1", u),
                            ped_s2=I("ped_s2", u), heg_s1=I("heg_s1", u), heg_s2=I("heg_s2", u))
    r.alice = [tuple(I(f, x, u) for f in ("alice_alpha", "alice_beta", "alice_gamma", "alice_rho")) for x in range(P)]
    for f in ("beta_tag_gamma", "r_gamma", "nonce_gamma_b", "nonce_gamma_beta", "beta_tag_w", "r_w", "nonce_w_b", "nonce_w_beta"):
        setattr(r, f, [I(f, j, u) for j in range(T - 1)])
    r.pdl = [tuple(I(f, j, u) for f in ("pdl_alpha", "pdl_beta", "pdl_rho", "pdl_gamma")) for j in range(T - 1)]
    return r


def _pt(row):
    v = int.from_bytes(np.ascontiguousarray(row).tobytes(), "little")
    return None if v == 0 else (v & ((1 << 256) - 1), v >> 256)


def _sc(row):
    return int.from_bytes(np.ascontiguousarray(row).tobytes(), "little")


def _oracle_sessions(jobs):
    """gen.offline_session over (keys, s_l, randomness) jobs, one process per session (the oracle's Paillier arithmetic is pure Python)"""
    import multiprocessing
    import os
    from concurrent.futures import ProcessPoolExecutor
    if len(jobs) < 2:
        return [gen.offline_session(*j) for j in jobs]
    with ProcessPoolExecutor(max_workers=min(len(jobs), os.cpu_count() or 1), mp_context=multiprocessing.get_context("spawn")) as pool:
        return list(pool.map(gen.offline_session, *zip(*jobs)))


def _check_against_oracle(out, keysets, sessions, inp, T, P):
    inp = {f: _host(v) for f, v in inp.items()}
    out = {f: _host(v) for f, v in out.items()}
    jobs = [([keysets[d[0]][i] for i in d[1:]], [i + 1 for i in d[1:]], [_party(inp, s * T + p, T, P) for p in range(T)]) for s, d in enumerate(sessions)]
    for s, (d, want) in enumerate(zip(sessions, _oracle_sessions(jobs))):
        s_l = [i + 1 for i in d[1:]]
        complete = all(wv.status == 0 for wv in want)
        assert int(out["complete"][s]) == int(complete)
        for p, wv in enumerate(want):
            u = s * T + p
            assert int(out["status"][u]) == wv.status, (s_l, p)
            if complete:
                assert (_pt(out["R"][u]), _sc(out["sigma"][u]), _sc(inp["k"][u]) % Q, _pt(out["T"][u])) == (wv.R, wv.sigma_i, wv.k_i, wv.t_vec[p]), (s_l, p)
            else:                       # a session that stopped produces nothing
                assert not out["R"][u].any() and not out["sigma"][u].any() and not out["T"][u].any()


@pytest.mark.parametrize("t,n,sets", [(1, 2, [[0, 1]]), (1, 3, [[2, 0], [1, 2, 0]]), (2, 5, [[4, 1, 2], [0, 1, 2, 3, 4]]), (3, 4, [[0, 1, 2, 3]]),
                                      (4, 8, [[7, 0, 3, 5, 1]])])
def test_parity_with_oracle(engine, t, n, sets):
    """one call per signing-set size, two key sets per call (fixture rows, and keys_edge.json rows where there are enough of them)"""
    from mpecdsa_b200 import gg20, gg20_general
    rng = random.Random(0x6E00 + 16 * t + n)
    fix, edge = _rows(), _rows(edge=True)
    keysets = [_key(fix[:n], t, n, rng), _key(edge[:n] if n <= len(edge) else fix[n:2 * n], t, n, rng)]
    ks = gg20.KeySets(engine, keysets)
    try:
        for s_l in sets:
            T = len(s_l)
            sessions = [[0] + s_l, [1] + s_l[::-1]]
            inp = gg20_general.sample_inputs(engine, ks, T, sessions, seed=SEED)
            out = gg20_general.offline_device(engine, ks, T, sessions, inp)
            assert list(out["complete"]) == [1, 1]
            _check_against_oracle(out, keysets, sessions, inp, T, n)
            print(f"({t}, {n}, {s_l}): two sessions equal the oracle", flush=True)
    finally:
        ks.free()


def _rnd_of(inp, T, E):
    """the arrays of sample_inputs as the `rnd` dict of gg20_general.offline_batch"""
    h = {f: _host(v) for f, v in inp.items()}
    ints = lambda a: [int.from_bytes(r.tobytes(), "little") for r in np.ascontiguousarray(a).reshape(-1, a.shape[-1])]
    rnd = {f: ints(h[f]) for f in ("gamma", "k", "blind", "r_k", "l", "ped_s1", "ped_s2", "heg_s1", "heg_s2")}
    al = [ints(h[f]) for f in ("alice_alpha", "alice_beta", "alice_gamma", "alice_rho")]
    P = h["alice_alpha"].shape[0]
    rnd["alice"] = [[tuple(a[x * E + u] for a in al) for x in range(P)] for u in range(E)]
    for f in ("beta_tag_gamma", "r_gamma", "nonce_gamma_b", "nonce_gamma_beta", "beta_tag_w", "r_w", "nonce_w_b", "nonce_w_beta"):
        v = ints(h[f])
        rnd[f] = [v[j * E + u] for u in range(E) for j in range(T - 1)]
    pd = [ints(h[f]) for f in ("pdl_alpha", "pdl_beta", "pdl_rho", "pdl_gamma")]
    rnd["pdl"] = [tuple(a[j * E + u] for a in pd) for u in range(E) for j in range(T - 1)]
    return rnd


def _driver_args(keysets, sessions, T, P):
    key_rows, all_rows, w, g_w, y = [], [], [], [], []
    for d in sessions:
        l_s = list(d[1:])
        for p in range(T):
            lk = keysets[d[0]][l_s[p]]
            lam = o.lagrange_at_zero(l_s[p], l_s)
            key_rows.append(d[0] * P + l_s[p]); all_rows.append([d[0] * P + x for x in range(P)])
            w.append(lam * lk.x_i % Q); g_w.append(o.pt_mul(lk.pk_vec[l_s[p]], lam)); y.append(lk.y_sum_s)
    return key_rows, all_rows, w, g_w, y


def test_equals_python_driver_and_fused_call_on_64_sessions(engine, pkg):
    """64 two-signer (1, 3) sessions over all fixture key sets: every output equals gg20_general.offline_batch on the same inputs and
    the fused tecdsa_gg20_offline_batch on the same values packed into TECDSA_RND_* records; the sampled inputs equal sample_rnd's;
    the one call executes fewer multiply-accumulates than the Python driver (each MessageA's range proofs verified once)"""
    from mpecdsa_b200 import gg20, gg20_general
    keysets = fixtures.load_all_keysets()
    ks = gg20.KeySets(engine, keysets)
    rng = random.Random(0x64)
    sessions = [[s % len(keysets)] + rng.sample(range(3), 2) for s in range(64)]
    T, E = 2, 128
    try:
        inp = gg20_general.sample_inputs(engine, ks, T, sessions, seed=SEED)
        key_rows, all_rows, w, g_w, y = _driver_args(keysets, sessions, T, 3)
        rnd = gg20_general.sample_rnd(engine, ks, T, key_rows, all_rows, seed=SEED)
        assert rnd == _rnd_of(inp, T, E)
        engine.work(reset=True)
        out = gg20_general.offline_device(engine, ks, T, sessions, inp)
        one_call = engine.work(reset=True)
        ref = gg20_general.offline_batch(engine, ks, T, key_rows, all_rows, w, g_w, y, rnd)
        driver = engine.work(reset=True)
        assert 0 < one_call < driver
        assert list(out["status"]) == list(ref["status"]) == [0] * E and list(out["complete"]) == [1] * 64
        for u in range(E):
            assert (_pt(out["R"][u]), _sc(out["sigma"][u]), _pt(out["T"][u])) == (ref["R"][u], ref["sigma"][u], ref["T"][u]), u
        # the fused two-signer call on the same values
        units = []
        for u in range(E):
            r = _party(inp, u, T, 3)
            units.append(o.UnitRandomness(gamma_i=r.gamma_i, k_i=r.k_i, blind=r.blind, r_k=r.r_k, alice=r.alice, beta_tag_gamma=r.beta_tag_gamma[0],
                                          r_gamma=r.r_gamma[0], nonce_gamma_b=r.nonce_gamma_b[0], nonce_gamma_beta=r.nonce_gamma_beta[0],
                                          beta_tag_w=r.beta_tag_w[0], r_w=r.r_w[0], nonce_w_b=r.nonce_w_b[0], nonce_w_beta=r.nonce_w_beta[0], l=r.l,
                                          ped_s1=r.ped_s1, ped_s2=r.ped_s2, pdl=r.pdl[0], heg_s1=r.heg_s1, heg_s2=r.heg_s2))
        fused = gg20.offline_batch(engine, ks, sessions, gg20.pack_randomness(units))
        assert (fused.status == out["status"]).all() and (fused.R == out["R"]).all() and (fused.sigma == out["sigma"]).all()
        for u in range(E):
            assert (fused.t_vec[u].reshape(2, 16)[u % 2] == out["T"][u]).all()
    finally:
        ks.free()


def test_failure_paths(engine, pkg):
    """a wrong x_i row fails its peers in round 2 and zeroes its session only; signers <= t ends in Phase6 for everyone; bad
    descriptors and bad mem are refused with every output at its sentinel"""
    from mpecdsa_b200 import gg20, gg20_general
    rng = random.Random(0xFA11)
    fix = _rows()
    key5 = _key(fix[:5], 2, 5, rng)
    bad = list(key5)
    import dataclasses
    bad[1] = dataclasses.replace(key5[1], x_i=(key5[1].x_i + 1) % Q)
    ks = gg20.KeySets(engine, [key5, bad])
    try:
        sessions = [[0, 4, 1, 2], [1, 4, 1, 2], [1, 0, 3, 4]]
        inp = gg20_general.sample_inputs(engine, ks, 3, sessions, seed=SEED)
        out = gg20_general.offline_device(engine, ks, 3, sessions, inp)
        assert list(out["status"]) == [0, 0, 0, pkg.ST_INVALID_KEY, 0, pkg.ST_INVALID_KEY, 0, 0, 0] and list(out["complete"]) == [1, 0, 1]
        assert not out["R"][3:6].any() and not out["sigma"][3:6].any() and not out["T"][3:6].any() and out["R"][6:].any(axis=1).all()
        _check_against_oracle(out, [key5, bad], sessions, inp, 3, 5)
        # two signers of a t = 2 key: the shares do not interpolate the key, so sum S != y in round 6 (Phase6Error)
        two = [[0, 0, 3]]
        inp2 = gg20_general.sample_inputs(engine, ks, 2, two, seed=SEED)
        out2 = gg20_general.offline_device(engine, ks, 2, two, inp2)
        assert list(out2["status"]) == [pkg.ST_PHASE6] * 2 and list(out2["complete"]) == [0]
        _check_against_oracle(out2, [key5, bad], two, inp2, 2, 5)
        # refused descriptors: key set out of range, index >= parties, repeated index, signers < 2, signers > parties; bad mem
        for T, d in ((3, [[2, 0, 1, 2]]), (3, [[0, 0, 1, 5]]), (3, [[0, 1, 3, 1]])):
            res = {"status": np.full(3, 0xEE, np.uint8), "R": np.full((3, 16), 0xEE, np.uint32), "sigma": np.full((3, 8), 0xEE, np.uint32),
                   "T": np.full((3, 16), 0xEE, np.uint32), "complete": np.full(1, 0xEE, np.uint8)}
            assert gg20_general.offline_device(engine, ks, T, d, inp, out=res, check=False) == -1
            assert all((v == 0xEE).all() for v in res.values())
        for T, d in ((1, [[0, 1]]), (6, [[0, 0, 1, 2, 3, 4, 0]])):
            res = {"status": np.full(T, 0xEE, np.uint8), "R": np.full((T, 16), 0xEE, np.uint32), "sigma": np.full((T, 8), 0xEE, np.uint32),
                   "T": np.full((T, 16), 0xEE, np.uint32), "complete": np.full(1, 0xEE, np.uint8)}
            assert gg20_general.offline_device(engine, ks, T, d, inp, out=res, check=False) == -1
            assert all((v == 0xEE).all() for v in res.values())
        for mem in (2, -1):
            assert gg20_general.offline_device(engine, ks, 3, np.array(sessions, np.uint32), inp, mem=mem, out=res, check=False) == -1
    finally:
        ks.free()


def test_device_buffers_equal_host(engine):
    """sample_inputs(DEVICE) equals the HOST draw, and offline_device on CUDA tensors writes exactly the HOST outputs"""
    import torch
    from mpecdsa_b200 import DEVICE, gg20, gg20_general
    rng = random.Random(0xDE7)
    fix = _rows()
    keysets = [_key(fix[:4], 2, 4, rng), _key(fix[4:8], 2, 4, rng)]
    ks = gg20.KeySets(engine, keysets)
    try:
        sessions = [[0, 3, 0, 1], [1, 2, 1, 3], [0, 0, 1, 2]]
        h_in = gg20_general.sample_inputs(engine, ks, 3, sessions, seed=SEED)
        d_sess = torch.tensor(sessions, dtype=torch.int32, device="cuda")
        d_in = gg20_general.sample_inputs(engine, ks, 3, d_sess, seed=SEED, mem=DEVICE)
        for f in h_in:
            assert (h_in[f] == _host(d_in[f])).all(), f
        h_out = gg20_general.offline_device(engine, ks, 3, sessions, h_in)
        d_out = gg20_general.offline_device(engine, ks, 3, d_sess, d_in, mem=DEVICE)
        torch.cuda.synchronize()
        for f in h_out:
            assert h_out[f].tobytes() == _host(d_out[f]).tobytes(), f
        assert list(h_out["complete"]) == [1, 1, 1]
    finally:
        ks.free()


def test_key_sets_of_any_size(engine, pkg):
    """tecdsa_keys_upload_parties(3) builds the tables tecdsa_keys_upload builds; KeySets refuses mixed sizes; a 5-party key set is
    refused by the four three-party calls"""
    import ctypes
    from mpecdsa_b200 import gg20
    keysets = fixtures.load_all_keysets()[:2]
    a = gg20.KeySets(engine, keysets)
    b = gg20.KeySets.__new__(gg20.KeySets)
    b.__dict__.update(a.__dict__)
    b.handle = ctypes.c_void_p()
    k = gg20._Keys(a.n, *[a._bufs[n].ctypes.data for n in ("paillier_p", "paillier_q", "n_tilde", "h1", "h2", "x_i", "pk", "y")])
    engine._ck(engine.lib.tecdsa_keys_upload_parties(engine._ctx, 3, ctypes.byref(k), ctypes.byref(b.handle)), "keys_upload_parties")
    try:
        for table, limbs in ((0, 64), (1, 128), (2, 64), (5, 64), (6, 64)):
            assert a.table(table, limbs) == b.table(table, limbs)
    finally:
        a.free(); b.free()
    with pytest.raises(ValueError):
        gg20.KeySets(engine, [keysets[0], keysets[1][:2]])
    rng = random.Random(5)
    ks5 = gg20.KeySets(engine, [_key(_rows()[:5], 2, 5, rng)])
    try:
        lib, sess = engine.lib, np.array([[0, 0, 1]], np.uint32)
        rnd = np.zeros((2, gg20.RND_LIMBS), np.uint32)
        z, st = np.zeros((2, 64), np.uint32), np.zeros(2, np.uint8)
        rec = np.zeros(2 * 256, np.uint8)
        sw = pkg.seed_words(SEED)
        assert lib.tecdsa_gg20_offline_batch(engine._ctx, ks5.handle, sess.ctypes.data, 1, rnd.ctypes.data, st.ctypes.data, None, None, None, None, 0) == -1
        lib.tecdsa_gg20_sample_randomness.argtypes = [ctypes.c_void_p] * 4 + [ctypes.c_void_p, ctypes.c_uint64, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int]
        assert lib.tecdsa_gg20_sample_randomness(engine._ctx, ks5.handle, sess.ctypes.data, 1, sw.ctypes.data, 0, rnd.ctypes.data, st.ctypes.data, 0) == -1
        lib.tecdsa_gg20_offline_records.argtypes = [ctypes.c_void_p] * 4 + [ctypes.c_size_t, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int]
        assert lib.tecdsa_gg20_offline_records(engine._ctx, ks5.handle, None, sess.ctypes.data, 1, rnd.ctypes.data, rec.ctypes.data, 0) == -1
        lib.tecdsa_gg20_sign_batch.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t] + [ctypes.c_void_p] * 9 + [ctypes.c_int]
        assert lib.tecdsa_gg20_sign_batch(engine._ctx, ks5.handle, sess.ctypes.data, 1, z.ctypes.data, z.ctypes.data, z.ctypes.data, z.ctypes.data, None,
                                          z.ctypes.data, z.ctypes.data, st.ctypes.data, st.ctypes.data, 0) == -1
        assert (rnd == 0).all() and (z == 0).all() and (rec == 0).all()
    finally:
        ks5.free()


def test_keygen_to_signatures_in_one_device_path(engine, pkg):
    """keygen_batch (2, 5) and (1, 3) -> KeySets of n-party key sets -> sample_inputs(DEVICE) -> offline_device -> sign_batch, and
    every signature verifies under OpenSSL against y_sum_s"""
    import torch
    from cryptography.hazmat.primitives import hashes
    from cryptography.hazmat.primitives.asymmetric import ec, utils
    from mpecdsa_b200 import DEVICE, gg20, gg20_general
    from tests import test_gg20_keygen_gpu as kgpu

    for t, n, s_l, seed in ((2, 5, [4, 1, 2], 0x7305), (1, 3, [2, 0], 0x7303)):
        primes = kgpu._primes(n, 2)
        res = kgpu._run(engine, t, n, primes, kgpu._inputs(t, n, primes, seed))
        assert list(res.complete) == [1, 1]
        keysets = [res.keys[0:n], res.keys[n:2 * n]]
        ks = gg20.KeySets(engine, keysets)
        try:
            T = len(s_l)
            sessions = torch.tensor([[0] + s_l, [1] + s_l[::-1]], dtype=torch.int32, device="cuda")
            inp = gg20_general.sample_inputs(engine, ks, T, sessions, seed=SEED, mem=DEVICE)
            out = gg20_general.offline_device(engine, ks, T, sessions, inp, mem=DEVICE)
            assert _host(out["complete"]).tolist() == [1, 1]
            msg = [random.Random(seed + s).getrandbits(256) % Q for s in range(2)]
            y = [keysets[0][0].y_sum_s, keysets[1][0].y_sum_s]
            sig = gg20_general.sign_batch(engine, T, msg, _host(out["R"]), _host(out["sigma"]), _host(inp["k"]), y)
            assert not sig["status"].any()
            for s in range(2):
                r_, s_ = _sc(sig["r"][s * T]), _sc(sig["s"][s * T])
                pub = ec.EllipticCurvePublicNumbers(y[s][0], y[s][1], ec.SECP256K1()).public_key()
                pub.verify(utils.encode_dss_signature(r_, s_), msg[s].to_bytes(32, "big"), ec.ECDSA(utils.Prehashed(hashes.SHA256())))
        finally:
            ks.free()
