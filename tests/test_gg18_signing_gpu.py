"""GPU tests of GG18 signing as one call (tecdsa_gg18_signing_batch): parity with the party-by-party restatement
(tests/gg18_signing_oracle.py) at (1, 3) / 2, (2, 5) / 3 and (4, 8) / 5 over fixture and keys_edge.json Paillier material, with every
signature accepted by OpenSSL; equality with gg18.sign_batch on 64 sessions of the same inputs, failing sessions included; the
failure paths and the isolation of failing sessions; refused arguments; DEVICE against HOST buffers; the sampled inputs against their
CPU restatement; and keys from tecdsa_gg20_keygen_batch through to signatures OpenSSL accepts."""
import dataclasses
import random

import numpy as np
import pytest

from oracle import gg20_oracle as o
from tests import gg18_signing_oracle as so
from tests.golden import fixtures

Q, G = o.Q, o.G
SEED = bytes(range(100, 132))
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


def _int(row):
    return int.from_bytes(np.ascontiguousarray(row).tobytes(), "little")


def _pt(row):
    v = _int(row)
    return None if v == 0 else (v & ((1 << 256) - 1), v >> 256)


def _signer(inp, u, T):
    r = so.SignerRandomness(**{f: _int(inp[f][u]) for f in so.ELEMENT_FIELDS})
    for f in so.PAIR_FIELDS:
        setattr(r, f, [_int(inp[f][j][u]) for j in range(T - 1)])
    return r


def _oracle(keysets, sessions, inp, messages, T):
    """so.sign_session per session, one process per session (the restatement's Paillier arithmetic is pure Python)"""
    import multiprocessing
    import os
    from concurrent.futures import ProcessPoolExecutor
    inp = {f: _host(v) for f, v in inp.items()}
    jobs = [([keysets[d[0]][i] for i in d[1:]], [i + 1 for i in d[1:]], [_signer(inp, s * T + p, T) for p in range(T)], messages[s])
            for s, d in enumerate(sessions)]
    if len(jobs) < 2:
        return [so.sign_session(*j) for j in jobs]
    with ProcessPoolExecutor(max_workers=min(len(jobs), os.cpu_count() or 1), mp_context=multiprocessing.get_context("spawn")) as pool:
        return list(pool.map(so.sign_session, *zip(*jobs)))


def _openssl_verify(y, r, s, m):
    from cryptography.hazmat.primitives import hashes
    from cryptography.hazmat.primitives.asymmetric import ec, utils
    pub = ec.EllipticCurvePublicNumbers(y[0], y[1], ec.SECP256K1()).public_key()
    pub.verify(utils.encode_dss_signature(r, s), m.to_bytes(32, "big"), ec.ECDSA(utils.Prehashed(hashes.SHA256())))


def _check_against_oracle(out, keysets, sessions, inp, messages, T):
    out = {f: _host(v) for f, v in out.items()}
    for s, (d, want) in enumerate(zip(sessions, _oracle(keysets, sessions, inp, messages, T))):
        assert out["status"][s * T:(s + 1) * T].tolist() == want.status, (s, d)
        assert int(out["complete"][s]) == int(want.signature is not None)
        for p in range(T):
            assert _pt(out["R"][s * T + p]) == want.R[p], (s, p)
        if want.signature:
            assert (_int(out["r"][s]), _int(out["s"][s]), int(out["recid"][s])) == want.signature
            _openssl_verify(keysets[d[0]][0].y_sum_s, _int(out["r"][s]), _int(out["s"][s]), messages[s])
        else:
            assert not out["r"][s].any() and not out["s"][s].any() and out["recid"][s] == 0


def _messages(n, seed):
    rng = random.Random(seed)
    return [rng.getrandbits(256) % Q for _ in range(n)]


@pytest.mark.parametrize("t,n,s_l", [(1, 3, [2, 0]), (2, 5, [4, 1, 2]), (4, 8, [7, 0, 3, 5, 1])])
def test_parity_with_oracle(engine, t, n, s_l):
    """one call of two sessions, one per key set (fixture rows, and keys_edge.json rows where there are enough of them)"""
    from mpecdsa_b200 import gg18, gg20
    rng = random.Random(0x1800 + 16 * t + n)
    fix, edge = _rows(), _rows(edge=True)
    keysets = [_key(fix[:n], t, n, rng), _key(edge[:n] if n <= len(edge) else fix[n:2 * n], t, n, rng)]
    ks = gg20.KeySets(engine, keysets)
    try:
        T = len(s_l)
        sessions = [[0] + s_l, [1] + s_l[::-1]]
        msg = _messages(2, t * 100 + n)
        inp = gg18.sample_inputs(engine, ks, T, sessions, seed=SEED)
        out = gg18.sign_device(engine, ks, T, sessions, msg, inp)
        assert list(out["complete"]) == [1, 1] and not out["status"].any()
        _check_against_oracle(out, keysets, sessions, inp, msg, T)
    finally:
        ks.free()


def _slice(inp, kept, T):
    """the inputs of the sessions `kept` of a batch, as a batch of their own"""
    idx = [s * T + p for s in kept for p in range(T)]
    return {f: np.ascontiguousarray(v[idx] if v.ndim == 2 else v[:, idx]) for f, v in inp.items()}


def _slice_out(out, kept, T):
    idx = [s * T + p for s in kept for p in range(T)]
    return {f: v[idx] if f in ("status", "R") else v[kept] for f, v in out.items()}


def _sign_batch_args(keysets, sessions, T, P, inp, msg):
    """the inputs of one call as the arguments of gg18.sign_batch (pair u * (T - 1) + j = alice u, bob ind(u, j))"""
    h = {f: _host(v) for f, v in inp.items()}
    E = len(sessions) * T
    key_rows, w, y, m = [], [], [], []
    for s, d in enumerate(sessions):
        l_s = list(d[1:])
        for p in range(T):
            lk = keysets[d[0]][l_s[p]]
            key_rows.append(d[0] * P + l_s[p]); w.append(o.lagrange_at_zero(l_s[p], l_s) * lk.x_i % Q); y.append(lk.y_sum_s); m.append(msg[s])
    rnd = {f: [_int(h[f][u]) for u in range(E)] for f in so.ELEMENT_FIELDS}
    names = {"r_b_gamma": "r_gamma", "beta_tag_gamma": "beta_tag_gamma", "r_b_w": "r_w", "beta_tag_w": "beta_tag_w", "nb_gamma": "nonce_gamma_b",
             "nbt_gamma": "nonce_gamma_beta", "nb_w": "nonce_w_b", "nbt_w": "nonce_w_beta"}
    for name, f in names.items():
        rnd[name] = []
        for u in range(E):
            for j in range(T - 1):
                pu = u % T
                pv = j if j < pu else j + 1
                v = u - pu + pv                                   # bob v answers alice u from its slab jb
                rnd[name].append(_int(h[f][pu if pu < pv else pu - 1][v]))
    return key_rows, w, y, m, rnd


def test_equals_sign_batch_on_64_sessions(engine, pkg):
    """64 two-signer sessions over all fixture key sets, three of them failing (a zero l in phase 5a, a zero delta sum in phase 3, a
    zero DLog nonce): a complete session equals gg18.sign_batch output for output; in a failing session the elements that carry a
    code carry sign_batch's, and the rest are OK"""
    import torch
    from mpecdsa_b200 import DEVICE, gg18, gg20
    keysets = fixtures.load_all_keysets()
    ks = gg20.KeySets(engine, keysets)
    rng = random.Random(0x6418)
    sessions = [[s % len(keysets)] + rng.sample(range(3), 2) for s in range(64)]
    T, E = 2, 128
    msg = _messages(64, 0x64)
    try:
        inp = gg18.sample_inputs(engine, ks, T, sessions, seed=SEED)
        inp["l"][5 * T + 1] = 0
        inp["gamma"][9 * T + 1] = np.frombuffer(((-_int(inp["gamma"][9 * T])) % Q).to_bytes(32, "little"), np.uint32)
        inp["dlog_nonce"][40 * T] = 0
        engine.work(reset=True)
        out = gg18.sign_device(engine, ks, T, sessions, msg, inp)
        one_call = engine.work(reset=True)
        key_rows, w, y, m, rnd = _sign_batch_args(keysets, sessions, T, 3, inp, msg)
        ref = gg18.sign_batch(engine, ks, T, key_rows, w, y, m, rnd)
        driver = engine.work(reset=True)
        print(f"executed MAC32: one call {one_call}, sign_batch {driver}")
        failing = {5: [0, pkg.ST_INVALID_KEY], 9: [pkg.ST_NOT_INVERTIBLE] * 2, 40: [pkg.ST_INVALID_KEY, 0]}
        assert [s for s in range(64) if not out["complete"][s]] == sorted(failing)
        for s in range(64):
            st = out["status"][s * T:(s + 1) * T].tolist()
            if s in failing:
                assert st == failing[s]
                for p in range(T):
                    if st[p]:
                        assert st[p] == ref["status"][s * T + p]
                assert not out["R"][s * T:(s + 1) * T].any() and not out["r"][s].any() and not out["s"][s].any()
                continue
            assert st == [0, 0] and not ref["status"][s * T:(s + 1) * T].any()
            for p in range(T):
                u = s * T + p
                assert _pt(out["R"][u]) == ref["R"][u]
                assert (_int(out["r"][s]), _int(out["s"][s]), int(out["recid"][s])) == (ref["r"][u], ref["s"][u], int(ref["recid"][u]))
        bad_s = sorted(failing)
        _check_against_oracle(_slice_out(out, bad_s, T), keysets, [sessions[s] for s in bad_s], _slice(inp, bad_s, T), [msg[s] for s in bad_s], T)
        # the same call on device buffers writes the same bytes
        d_sess = torch.tensor(sessions, dtype=torch.int32, device="cuda")
        d_in = gg18.sample_inputs(engine, ks, T, d_sess, seed=SEED, mem=DEVICE)
        h_in = gg18.sample_inputs(engine, ks, T, sessions, seed=SEED)
        for f in h_in:
            assert (h_in[f] == _host(d_in[f])).all(), f
        h_out = gg18.sign_device(engine, ks, T, sessions, msg, h_in)
        d_msg = torch.from_numpy(pkg.ints_to_limbs(msg, 8).view(np.int32)).cuda()
        d_out = gg18.sign_device(engine, ks, T, d_sess, d_msg, d_in, mem=DEVICE)
        torch.cuda.synchronize()
        for f in h_out:
            assert h_out[f].tobytes() == _host(d_out[f]).tobytes(), f
        assert list(h_out["complete"]) == [1] * 64
    finally:
        ks.free()


def test_failure_paths(engine, pkg):
    """a perturbed x_i row fails every member in 5d; a zero l, rho or DLog nonce fails its element in 5a; a zero delta sum fails every
    member in phase 3 — each against the oracle, and the other sessions' bytes equal a batch without the failing ones.  Refused
    descriptors, sizes, buffers and mem return TECDSA_E_ARG before any launch, with every output at its sentinel"""
    from mpecdsa_b200 import gg18, gg20
    rng = random.Random(0xFA18)
    fix = _rows()
    key5 = _key(fix[:5], 2, 5, rng)
    bad = list(key5)
    bad[1] = dataclasses.replace(key5[1], x_i=(key5[1].x_i + 1) % Q)
    ks = gg20.KeySets(engine, [key5, bad])
    T = 3
    try:
        sessions = [[0, 4, 1, 2], [1, 4, 1, 2], [0, 0, 3, 4], [0, 2, 3, 1], [0, 1, 0, 2], [1, 1, 0, 2], [0, 4, 3, 2]]
        n = len(sessions)
        msg = _messages(n, 0xFA)
        inp = gg18.sample_inputs(engine, ks, T, sessions, seed=SEED)
        inp["l"][2 * T + 1] = 0                                                   # session 2: 5a
        inp["rho"][3 * T + 2] = 0                                                 # session 3: 5a
        inp["dlog_nonce"][4 * T] = 0                                              # session 4: 5a
        inp["gamma"][6 * T + 2] = np.frombuffer(((-(_int(inp["gamma"][6 * T]) + _int(inp["gamma"][6 * T + 1]))) % Q).to_bytes(32, "little"), np.uint32)
        out = gg18.sign_device(engine, ks, T, sessions, msg, inp)
        IK, NI = pkg.ST_INVALID_KEY, pkg.ST_NOT_INVERTIBLE
        assert out["status"].reshape(n, T).tolist() == [[0] * 3, [IK] * 3, [0, IK, 0], [0, 0, IK], [IK, 0, 0], [IK] * 3, [NI] * 3]
        assert list(out["complete"]) == [1, 0, 0, 0, 0, 0, 0]
        _check_against_oracle(out, [key5, bad], sessions, inp, msg, T)
        # the failing sessions do not disturb the others: session 0 alone gives the same bytes
        alone = gg18.sign_device(engine, ks, T, [sessions[0]], msg[:1], _slice(inp, [0], T))
        assert alone["status"].tobytes() == out["status"][:T].tobytes() and alone["R"].tobytes() == out["R"][:T].tobytes()
        assert alone["r"].tobytes() == out["r"][:1].tobytes() and alone["s"].tobytes() == out["s"][:1].tobytes()
        # refused calls touch nothing and launch nothing
        def refused(T_, d, m, inp_, mem=pkg.HOST):
            k = len(d) * T_
            res = {"status": np.full(k, 0xEE, np.uint8), "R": np.full((k, 16), 0xEE, np.uint32), "sig_r": np.full((len(d), 8), 0xEE, np.uint32),
                   "sig_s": np.full((len(d), 8), 0xEE, np.uint32), "recid": np.full(len(d), 0xEE, np.uint8), "complete": np.full(len(d), 0xEE, np.uint8)}
            before = engine.launch_count()
            rc = gg18.sign_device(engine, ks, T_, np.array(d, np.uint32), m, inp_, mem=mem, out=res, check=False)
            assert rc == -1 and engine.launch_count() == before
            assert all((v == 0xEE).all() for v in res.values())
        one = _slice(inp, [0], T)
        for d in ([[2, 0, 1, 2]], [[0, 0, 1, 5]], [[0, 1, 3, 1]]):            # key set out of range, index >= parties, repeated index
            refused(3, d, msg[:1], one)
        refused(1, [[0, 1]], msg[:1], one)                                        # signers < 2
        refused(6, [[0, 0, 1, 2, 3, 4, 0]], msg[:1], one)                          # signers > parties
        for f in ("rho", "nonce_w_beta"):                                         # a NULL buffer
            refused(3, [sessions[0]], msg[:1], {**one, f: None})
        for mem in (2, -1):                                                       # a bad mem
            refused(3, [sessions[0]], msg[:1], one, mem=mem)
        lib = engine.lib
        big = (1 << 24) + 1                                                        # an oversize batch (checked before the descriptors are read)
        from mpecdsa_b200.gg18 import _SigningIn, _SigningOut, IN_FIELDS, OUT_FIELDS
        import ctypes
        z = np.zeros(16, np.uint32)
        gi = _SigningIn(*[z.ctypes.data] * len(IN_FIELDS))
        go = _SigningOut(*[z.ctypes.data] * len(OUT_FIELDS))
        before = engine.launch_count()
        assert lib.tecdsa_gg18_signing_batch(engine._ctx, ks.handle, 3, big, 0, z.ctypes.data, z.ctypes.data, ctypes.byref(gi), ctypes.byref(go)) == -1
        assert lib.tecdsa_gg18_signing_batch(engine._ctx, ks.handle, 3, 0, 0, z.ctypes.data, z.ctypes.data, ctypes.byref(gi), ctypes.byref(go)) == 0
        assert engine.launch_count() == before and not z.any()
    finally:
        ks.free()


def test_sampler_equals_cpu_restatement(engine):
    """sample_inputs values equal gg18_signing_oracle.sample_inputs (ChaCha20 streams restated on the CPU) on a sample of elements"""
    from mpecdsa_b200 import gg18, gg20
    rng = random.Random(0x5A18)
    keysets = [_key(_rows()[:5], 2, 5, rng), _key(_rows()[5:10], 2, 5, rng)]
    ks = gg20.KeySets(engine, keysets)
    try:
        T, sessions = 4, [[1, 4, 0, 2, 3], [0, 1, 2, 3, 4], [1, 0, 1, 2, 3]]
        inp = gg18.sample_inputs(engine, ks, T, sessions, seed=SEED)
        N = ks.table(0, 64)
        want = so.sample_inputs(SEED, N, 5, T, sessions, elements=[0, 5, 11])
        for u, r in want.items():
            assert _signer(inp, u, T) == r, u
    finally:
        ks.free()


def test_keygen_to_signatures_in_one_device_path(engine, pkg):
    """keygen_batch (2, 5) and (1, 3) -> KeySets -> sample_inputs(DEVICE) -> sign_device(DEVICE) with three and two signers, and every
    signature verifies under OpenSSL against y_sum_s"""
    import torch
    from mpecdsa_b200 import DEVICE, gg18, gg20
    from tests import test_gg20_keygen_gpu as kgpu

    for t, n, s_l, seed in ((2, 5, [4, 1, 2], 0x7318), (1, 3, [2, 0], 0x7313)):
        primes = kgpu._primes(n, 2)
        res = kgpu._run(engine, t, n, primes, kgpu._inputs(t, n, primes, seed))
        assert list(res.complete) == [1, 1]
        keysets = [res.keys[0:n], res.keys[n:2 * n]]
        ks = gg20.KeySets(engine, keysets)
        try:
            T = len(s_l)
            sessions = torch.tensor([[0] + s_l, [1] + s_l[::-1]], dtype=torch.int32, device="cuda")
            msg = _messages(2, seed)
            inp = gg18.sample_inputs(engine, ks, T, sessions, seed=SEED, mem=DEVICE)
            d_msg = torch.from_numpy(pkg.ints_to_limbs(msg, 8).view(np.int32)).cuda()
            out = gg18.sign_device(engine, ks, T, sessions, d_msg, inp, mem=DEVICE)
            assert _host(out["complete"]).tolist() == [1, 1] and not _host(out["status"]).any()
            r, s = _host(out["r"]), _host(out["s"])
            for i in range(2):
                _openssl_verify(keysets[i][0].y_sum_s, _int(r[i]), _int(s[i]), msg[i])
        finally:
            ks.free()
