"""GPU tests of the one-call drivers at the edge of their declared domain: GG20 key generation at (t, n) = (63, 64) with every
output restated from its inputs, bad-actor masks with bits 32 and 63 at (1, 64) and (63, 64), the GG20 offline stage and GG18
signing with all 64 signers of those keys and with two signers at P = 64, wrong key shares at signer positions 32 and 63, and
refused oversize arguments.  Sessions too large for the party-by-party oracle are checked against the plain scalar reference of
their MtA shares (tests/test_domain_limits.py::mta_session) and OpenSSL."""
import ctypes
import dataclasses
import random

import numpy as np
import pytest

from oracle import gg20_oracle as o
from oracle import keygen_oracle as kg
from tests import keygen_group as kgg
from tests import test_gg20_keygen_gpu as kgpu
from tests.test_domain_limits import mta_session, signature
from tests.test_gg18_signing_gpu import _openssl_verify

pytestmark = pytest.mark.gpu
Q, G = o.Q, o.G
SEED = bytes(range(64, 96))
N64, T64 = 64, 63
IK = kgg.ST_INVALID_KEY
HIGH = (1 << 32) | (1 << 63)


def _int(row):
    return int.from_bytes(np.ascontiguousarray(row).tobytes(), "little")


def _pt(row):
    v = _int(row)
    return None if v == 0 else (v & ((1 << 256) - 1), v >> 256)


def _limbs(v, k):
    return np.frombuffer(int(v).to_bytes(4 * k, "little"), np.uint32)


def _primes64():
    """64 parties: the 64 distinct N~ pairs of tests/golden/n_tilde_64.json; the Paillier primes reuse the 12 fixture rows cyclically
    (a repeated N changes no per-party check of key generation, and the fixtures hold only 12 Paillier keys)"""
    import json
    import os
    with open(os.path.join(os.path.dirname(os.path.abspath(kgpu.fixtures.__file__)), "n_tilde_64.json")) as f:
        nt = [(int(p, 16), int(q, 16)) for p, q in json.load(f)["pairs"]]
    assert len(nt) == N64 and len({p for pr in nt for p in pr}) == 2 * N64
    assert all(p.bit_length() == q.bit_length() == 1024 and pow(2, p - 1, p) == 1 and pow(2, q - 1, q) == 1 for p, q in nt)
    rows = kgpu._rows()
    return [((rows[i % 12].dk.p, rows[i % 12].dk.q), nt[i]) for i in range(N64)]


def _mul_G(k):
    """k G for 0 < k < q through OpenSSL (thousands of them, too many for the oracle's pure-Python scalar multiplication)"""
    from cryptography.hazmat.primitives.asymmetric import ec
    pn = ec.derive_private_key(k, ec.SECP256K1()).public_key().public_numbers()
    return (pn.x, pn.y)


@pytest.fixture(scope="module")
def keygen64(engine):
    """one (63, 64) group through tecdsa_gg20_keygen_batch"""
    primes = _primes64()
    rnd = kgpu._inputs(T64, N64, primes, 0x6463)
    res = kgpu._run(engine, T64, N64, primes, rnd)
    assert list(res.complete) == [1]
    return primes, rnd, res


def _oracle_key(lk):
    """a LocalKey of the package as oracle.LocalKey (picklable into the oracle's worker processes)"""
    return o.LocalKey(i=lk.i, t=lk.t, n=lk.n, x_i=lk.x_i, dk=o.DecryptionKey(lk.dk.p, lk.dk.q), pk_vec=list(lk.pk_vec),
                      paillier_key_vec=[o.EncryptionKey(e.n, e.n * e.n) for e in lk.paillier_key_vec],
                      h1_h2_n_tilde_vec=[o.DLogStatement(s.N, s.g, s.ni) for s in lk.h1_h2_n_tilde_vec], y_sum_s=lk.y_sum_s)


@pytest.fixture(scope="module")
def keysets64(engine, keygen64):
    """KeySets of two 64-party key sets: the (63, 64) keys, and the same keys with a wrong x_i for party 33"""
    from mpecdsa_b200 import gg20
    keys = [_oracle_key(lk) for lk in keygen64[2].keys]
    bad = list(keys)
    bad[32] = dataclasses.replace(keys[32], x_i=(keys[32].x_i + 1) % Q)
    ks = gg20.KeySets(engine, [keys, bad])
    yield [keys, bad], ks
    ks.free()


def test_keygen_63_of_64(keygen64):
    """every output of a complete (63, 64) group restated from its inputs: x_i = sum_s f_s(i) from the sampled coefficients,
    pk_vec[j] = x_j G, y = (sum u_s) G, N = p q and (N~, h1, h2 = h1^xhi) of every party, commitment 0 of every party and all 64
    commitments f_i,k G of parties 1, 2, 33, 63 and 64; any 64 shares interpolate to sum u_s.  The party-by-party group oracle
    (tests/keygen_group.py) restates the same outputs through every proof, but at n = 64 it costs minutes of pure-Python curve
    arithmetic; its verdicts are checked at n <= 5 in test_gg20_keygen_gpu.py"""
    primes, rnd, res = keygen64
    polys = [[r["u"]] + list(r["coeffs"]) for r in rnd]
    f = lambda c, x: sum(a * pow(x, k, Q) for k, a in enumerate(c)) % Q
    x = [sum(f(c, i + 1) for c in polys) % Q for i in range(N64)]
    u = sum(c[0] for c in polys) % Q
    assert kgg.lagrange_at_zero([(i + 1, x[i]) for i in range(N64)]) == u
    pk, y = [_mul_G(v) for v in x], _mul_G(u)
    assert pk[32] == o.pt_mul(G, x[32]) and y == o.pt_mul(G, u)                     # the OpenSSL products against the oracle's
    ns = [p * q for (p, q), _ in primes]
    sts = [kg.h1_h2_n_tilde(pt, qt, r["h1"], r["xhi"])[:3] for (_, (pt, qt)), r in zip(primes, rnd)]
    assert list(res.status) == [kgg.ST_OK] * N64 and [int(b) for b in res.bad_actors] == [0] * N64
    for i, lk in enumerate(res.keys):
        assert (lk.i, lk.t, lk.n, lk.x_i, lk.dk.p, lk.dk.q) == (i + 1, T64, N64, x[i], *primes[i][0])
        assert lk.pk_vec == pk and lk.y_sum_s == y and [e.n for e in lk.paillier_key_vec] == ns
        assert [(s.N, s.g, s.ni) for s in lk.h1_h2_n_tilde_vec] == sts
        assert len(lk.vss_commitments) == T64 + 1 and lk.vss_commitments[0] == _mul_G(polys[i][0])
    for i in (0, 1, 32, 62, 63):
        assert res.keys[i].vss_commitments == [_mul_G(c) for c in polys[i]], i


@pytest.mark.parametrize("t", [1, T64])
def test_keygen_masks_with_bits_32_and_63(engine, keygen64, t):
    """parties 33 and 64 of the second group have a 2046-bit N: every element of that group is INVALID_KEY with the mask
    2^32 + 2^63 (read back as that integer) and no key; the first group is byte-identical to a call of its own"""
    primes, rnd, clean = keygen64
    if t != T64:
        rnd = kgpu._inputs(t, N64, primes, 0x6401)
        clean = kgpu._run(engine, t, N64, primes, rnd)
    assert list(clean.complete) == [1]
    p2 = list(primes)
    for i in (32, 63):
        (p, q), nt = p2[i]
        p2[i] = ((p >> 2 | 1, q), nt)
    res = kgpu._run(engine, t, N64, primes + p2, rnd + rnd)
    assert list(res.complete) == [1, 0]
    assert [int(b) for b in res.bad_actors[N64:]] == [HIGH] * N64 and list(res.status[N64:]) == [IK] * N64
    assert all(k is None for k in res.keys[N64:])
    for f, a in res.out.items():
        b = clean.out[f]
        per = a.shape[0] // 2
        assert np.array_equal(a[:per], b), f
        if f not in ("status", "bad_actors", "complete"):
            assert not a[per:].any(), f


def _set_bt(inp, field, T, s, alice, bob, value):
    """overwrite the beta' Bob (position) sends Alice (position) in session s"""
    j = alice if alice < bob else alice - 1
    inp[field][j][s * T + bob] = _limbs(value, 64)


def _reference(keysets, d, inp, T, s, gg18=False):
    keys = [keysets[d[0]][i] for i in d[1:]]
    u0 = s * T
    k = [_int(inp["k"][u0 + p]) for p in range(T)]
    g = [_int(inp["gamma"][u0 + p]) for p in range(T)]
    bt = {f: [[_int(inp[f][j][u0 + p]) for j in range(T - 1)] for p in range(T)] for f in ("beta_tag_gamma", "beta_tag_w")}
    l = None if gg18 else [_int(inp["l"][u0 + p]) for p in range(T)]
    return mta_session(keys, list(d[1:]), k, g, bt["beta_tag_gamma"], bt["beta_tag_w"], l), k


def _sessions64(rng):
    perm = rng.sample(range(N64), N64)
    to_end = [i for i in range(N64) if i != 32] + [32]                  # party 33 at position 63
    return perm, [[0] + list(range(N64)),                                # clean
                  [0] + perm,                                           # alice shares of zero on pairs >= 32
                  [0] + perm[::-1],                                     # a beta' of N_a - 1 on pair 62 -> 33
                  [1] + list(range(N64)),                               # wrong x_i at position 32
                  [1] + to_end]                                         # wrong x_i at position 63


def _overwrite(inp, keysets, sessions, T):
    """session 1: Alice's share is zero on (alice 40, bob 50) for gamma and (alice 63, bob 32) for w; session 2: beta' = N_a - 1 on
    (alice 33, bob 62) for gamma"""
    for a, b, f in ((40, 50, "beta_tag_gamma"), (63, 32, "beta_tag_w")):
        u_a, u_b = T + a, T + b
        k = _int(inp["k"][u_a]) % Q
        if f == "beta_tag_gamma":
            x = _int(inp["gamma"][u_b]) % Q
        else:
            l_s = sessions[1][1:]
            x = o.lagrange_at_zero(l_s[b], l_s) * keysets[0][l_s[b]].x_i % Q
        _set_bt(inp, f, T, 1, a, b, -k * x % Q)
    N = keysets[0][sessions[2][1 + 33]].paillier_key_vec[sessions[2][1 + 33]].n
    _set_bt(inp, "beta_tag_gamma", T, 2, 33, 62, N - 1)


def _expect(ref, T, tampered, gg18):
    """the statuses the oracles' rules give: a failed MessageB check stops its receiver (GG20 round 2, GG18 get_alpha); a wrong
    x_i fails every peer of its signer in GG20's round-2 key check, and every signer in GG18's phase 5d"""
    if any(ref.mta_bad):
        return [IK if m else 0 for m in ref.mta_bad]
    if tampered is not None:
        return [IK] * T if gg18 else [0 if p == tampered else IK for p in range(T)]
    return [0] * T


def test_offline_64_signers(engine, keysets64):
    """five 64-signer sessions in one call, checked element by element against the scalar reference: a clean one, one with zero
    Alice shares on pairs whose positions are >= 32, one with a wrapping beta', a wrong x_i at position 32 and at position 63; the
    clean session signs (OpenSSL accepts) and is byte-identical to a call of its own"""
    from mpecdsa_b200 import gg20_general
    keysets, ks = keysets64
    T = N64
    perm, sessions = _sessions64(random.Random(0x6420))
    inp = gg20_general.sample_inputs(engine, ks, T, sessions, seed=SEED)
    alone = gg20_general.offline_device(engine, ks, T, sessions[:1], {f: np.ascontiguousarray(v[..., :T, :]) for f, v in inp.items()})
    _overwrite(inp, keysets, sessions, T)
    out = gg20_general.offline_device(engine, ks, T, sessions, inp)
    assert list(out["complete"]) == [1, 1, 0, 0, 0]
    for s, d in enumerate(sessions):
        ref, k = _reference(keysets, d, inp, T, s)
        tampered = d[1:].index(32) if d[0] == 1 else None
        rows = slice(s * T, (s + 1) * T)
        assert out["status"][rows].tolist() == _expect(ref, T, tampered, False), s
        if ref.R is None:
            assert not out["R"][rows].any() and not out["sigma"][rows].any() and not out["T"][rows].any()
            continue
        for p in range(T):
            u = s * T + p
            assert (_pt(out["R"][u]), _int(out["sigma"][u]), _pt(out["T"][u])) == (ref.R, ref.sigma[p], ref.T[p]), (s, p)
        m = random.Random(s).getrandbits(256) % Q
        r_, s_, _ = signature(ref, k, m)
        _openssl_verify(keysets[0][0].y_sum_s, r_, s_, m)
    for f in alone:
        assert alone[f].tobytes() == out[f][:alone[f].shape[0]].tobytes(), f


def test_offline_two_signers_at_64_parties(engine, keysets64):
    """[63, 0], [0, 63] and [31, 32] of a (1, 64) key over the Paillier and N~ material of the keygen call (two signers of the
    (63, 64) key stop in round 6) in one call, with MessageA range proofs over statements x up to 63: every session completes and
    R, sigma_i and T_i equal the scalar reference"""
    from mpecdsa_b200 import gg20, gg20_general
    keysets, _ = keysets64
    rng = random.Random(0x6402)
    c0, c1 = rng.randrange(1, Q), rng.randrange(1, Q)
    x = [(c0 + c1 * (i + 1)) % Q for i in range(N64)]
    pks = [o.pt_mul(G, v) for v in x]
    keys1 = [dataclasses.replace(lk, t=1, x_i=x[i], pk_vec=pks, y_sum_s=o.pt_mul(G, c0)) for i, lk in enumerate(keysets[0])]
    ks = gg20.KeySets(engine, [keys1])
    try:
        sessions = [[0, 63, 0], [0, 0, 63], [0, 31, 32]]
        inp = gg20_general.sample_inputs(engine, ks, 2, sessions, seed=SEED)
        out = gg20_general.offline_device(engine, ks, 2, sessions, inp)
    finally:
        ks.free()
    assert list(out["complete"]) == [1, 1, 1]
    for s, d in enumerate(sessions):
        ref, _ = _reference([keys1], d, inp, 2, s)
        for p in range(2):
            assert (_pt(out["R"][2 * s + p]), _int(out["sigma"][2 * s + p]), _pt(out["T"][2 * s + p])) == (ref.R, ref.sigma[p], ref.T[p])


def test_gg18_wrong_share_pattern_at_5(engine, keysets64):
    """the restatement's verdict on a wrong x_i (every signer INVALID_KEY), on the device at T = 5 with party 33 among the signers"""
    from mpecdsa_b200 import gg18
    from tests.test_gg18_signing_gpu import _check_against_oracle as check18
    keysets, ks = keysets64
    sessions = [[1, 40, 32, 7, 63, 0]]
    msg = [random.Random(5).getrandbits(256) % Q]
    inp = gg18.sample_inputs(engine, ks, 5, sessions, seed=SEED)
    out = gg18.sign_device(engine, ks, 5, sessions, msg, inp)
    assert out["status"].tolist() == [IK] * 5 and list(out["complete"]) == [0]
    check18(out, keysets, sessions, inp, msg, 5)


def test_gg18_64_signers(engine, keysets64):
    """the five sessions of test_offline_64_signers through GG18 signing: R and the signature of the complete sessions equal the
    scalar reference and OpenSSL accepts them; the failing ones follow the restatement's rules; the clean session is byte-identical
    to a call of its own"""
    from mpecdsa_b200 import gg18
    keysets, ks = keysets64
    T = N64
    perm, sessions = _sessions64(random.Random(0x6418))
    msg = [random.Random(0x18 + s).getrandbits(256) % Q for s in range(len(sessions))]
    inp = gg18.sample_inputs(engine, ks, T, sessions, seed=SEED)
    alone = gg18.sign_device(engine, ks, T, sessions[:1], msg[:1], {f: np.ascontiguousarray(v[..., :T, :]) for f, v in inp.items()})
    _overwrite(inp, keysets, sessions, T)
    out = gg18.sign_device(engine, ks, T, sessions, msg, inp)
    assert list(out["complete"]) == [1, 1, 0, 0, 0]
    for s, d in enumerate(sessions):
        ref, k = _reference(keysets, d, inp, T, s, gg18=True)
        tampered = d[1:].index(32) if d[0] == 1 else None
        assert out["status"][s * T:(s + 1) * T].tolist() == _expect(ref, T, tampered, True), s
        if ref.R is None or tampered is not None:
            assert not out["R"][s * T:(s + 1) * T].any() and not out["r"][s].any() and not out["s"][s].any()
            continue
        assert all(_pt(out["R"][s * T + p]) == ref.R for p in range(T))
        want = signature(ref, k, msg[s])
        assert (_int(out["r"][s]), _int(out["s"][s]), int(out["recid"][s])) == want
        _openssl_verify(keysets[0][0].y_sum_s, want[0], want[1], msg[s])
    for f in alone:
        assert alone[f].tobytes() == out[f][:alone[f].shape[0]].tobytes(), f


def test_oversize_arguments_are_refused(engine, pkg, keysets64):
    """65 parties, keygen groups past the 32-bit job index at n = 64, and n_sessions * T * P = 2^26 + T * P at T = P = 64: each
    call returns TECDSA_E_ARG and launches nothing (no buffer that large is ever allocated)"""
    from mpecdsa_b200 import gg18, gg20, gg20_general, keygen
    keysets, ks = keysets64
    lib = engine.lib
    z = np.zeros(64, np.uint32)
    fx = gg20.KeySets(engine, kgpu.fixtures.load_all_keysets()[:1])
    try:
        k = gg20._Keys(fx.n, *[fx._bufs[f].ctypes.data for f in ("paillier_p", "paillier_q", "n_tilde", "h1", "h2", "x_i", "pk", "y")])
        handle = ctypes.c_void_p()
        before = engine.launch_count()
        assert lib.tecdsa_keys_upload_parties(engine._ctx, 65, ctypes.byref(k), ctypes.byref(handle)) == -1 and not handle.value
    finally:
        fx.free()
    V, S_, I_ = ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int
    lib.tecdsa_gg20_keygen_batch.argtypes = [V, I_, I_, S_, I_, ctypes.POINTER(keygen._KeygenIn), ctypes.POINTER(keygen._KeygenOut)]
    lib.tecdsa_gg20_offline_general_batch.argtypes = [V, V, I_, S_, I_, V, ctypes.POINTER(gg20_general._GeneralIn), ctypes.POINTER(gg20_general._GeneralOut)]
    gg18._bind(lib)
    groups = (2 ** 31 - 1) // 64 // (11 * 64) + 1
    kin = keygen._KeygenIn(*[z.ctypes.data] * len(keygen._KeygenIn._fields_))
    kout = keygen._KeygenOut(*[z.ctypes.data] * len(keygen._KeygenOut._fields_))
    n_sessions = (1 << 26) // (N64 * N64) + 1
    assert n_sessions * N64 * N64 == (1 << 26) + N64 * N64
    gin = gg20_general._GeneralIn(*[z.ctypes.data] * len(gg20_general.IN_FIELDS))
    gout = gg20_general._GeneralOut(*[z.ctypes.data] * 5)
    sin = gg18._SigningIn(*[z.ctypes.data] * len(gg18.IN_FIELDS))
    sout = gg18._SigningOut(*[z.ctypes.data] * len(gg18.OUT_FIELDS))
    assert lib.tecdsa_gg20_keygen_batch(engine._ctx, T64, N64, groups, pkg.HOST, ctypes.byref(kin), ctypes.byref(kout)) == -1
    assert lib.tecdsa_gg20_offline_general_batch(engine._ctx, ks.handle, N64, n_sessions, pkg.HOST, z.ctypes.data, ctypes.byref(gin), ctypes.byref(gout)) == -1
    assert lib.tecdsa_gg18_signing_batch(engine._ctx, ks.handle, N64, n_sessions, pkg.HOST, z.ctypes.data, z.ctypes.data, ctypes.byref(sin), ctypes.byref(sout)) == -1
    assert engine.launch_count() == before and not z.any()
