"""Other protocols on the same primitives (SURVEY.md section 8(f) rank 4): Lindell-2017 two-party ECDSA, the interactive PDL proof and
the GG18 phases 4 / 5a-5d.  CPU: the oracles' restatements run the reference's own test flows (`test_two_party_sign`,
`test_full_key_gen` of lindell_2017/test.rs, the phase-5 part of gg_2018/test.rs `sign`) and the final signatures verify under an
independent ECDSA (`cryptography`).  GPU: every new entry point against the oracle, bit for bit, plus tampered inputs, on the
standard key set and on the key sets of keys_edge.json, whose rows also carry inputs at the top of each sampling range."""
import random

import numpy as np
import pytest

from oracle import gg18_oracle as e18
from oracle import gg20_oracle as o
from oracle import keygen_oracle as kg
from oracle import lindell17_oracle as l17
from tests.golden import fixtures
from tests.golden.make_edge_keys import HALF, SLACK, prime_in
from tests.test_edge_keys import _worst_plaintexts

Q, G = o.Q, o.G


def _edge_rows():
    """(global key row, oracle.LocalKey, shape) of the 9 edge rows, in the order gg20.KeySets(engine, edge) uploads them"""
    shapes = [r["shape"] for ks in fixtures.edge_keysets_raw() for r in ks["parties"]]
    return [(i, lk, s) for i, (lk, s) in enumerate(zip([lk for ks in fixtures.load_edge_keysets() for lk in ks], shapes))]


def _ecdsa_ok(r, s, pub, msg_int):
    """independent check under OpenSSL: msg_int is the (already hashed) 256-bit message"""
    from cryptography.hazmat.primitives import hashes
    from cryptography.hazmat.primitives.asymmetric import ec, utils
    key = ec.EllipticCurvePublicNumbers(pub[0], pub[1], ec.SECP256K1()).public_key()
    try:
        key.verify(utils.encode_dss_signature(r, s), (msg_int % (1 << 256)).to_bytes(32, "big"), ec.ECDSA(utils.Prehashed(hashes.SHA256())))
        return True
    except Exception:
        return False


def _l17_case(keyset, rng, n):
    """n independent two-party signing instances under the Paillier keys of the key set (party one = key row i % 3)"""
    rows = [i % 3 for i in range(n)]
    dks = [keyset[r].dk for r in rows]
    eks = [o.EncryptionKey(d.p * d.q, (d.p * d.q) ** 2) for d in dks]
    c = dict(rows=rows, dks=dks, eks=eks)
    c["x1"] = [rng.randrange(1, Q // 3) for _ in range(n)]
    c["x2"] = [rng.randrange(1, Q) for _ in range(n)]
    c["r_key"] = [rng.randrange(1, ek.n) for ek in eks]
    c["c_key"] = [o.paillier_encrypt(ek, x, r) for ek, x, r in zip(eks, c["x1"], c["r_key"])]
    for name in ("k1", "k2", "n1", "n2"):
        c[name] = [rng.randrange(1, Q) for _ in range(n)]
    for name in ("b1", "b2"):
        c[name] = [rng.getrandbits(256) for _ in range(n)]
    c["msg"] = [rng.getrandbits(256) for _ in range(n)]
    c["rho"] = [rng.randrange(Q * Q) for _ in range(n)]
    c["r_enc"] = [rng.randrange(1, ek.n) for ek in eks]
    c["pub"] = [o.pt_mul(G, a * b % Q) for a, b in zip(c["x1"], c["x2"])]
    return c


def test_lindell17_oracle_flow(keyset):
    rng = random.Random(0x117)
    c = _l17_case(keyset, rng, 3)
    for i in range(3):
        # key generation messages (test_d_log_proof_party_two_party_one)
        first = l17.p1_keygen_first(c["x1"][i], c["n1"][i], c["b1"][i], c["b2"][i])
        assert l17.p2_keygen_verify(first, c["b1"][i], c["b2"][i])
        assert not l17.p2_keygen_verify(first, c["b1"][i] ^ 1, c["b2"][i])
        # ephemeral exchange + signature (test_two_party_sign)
        e1 = l17.eph_create(c["k1"][i], c["n1"][i])
        e2 = l17.eph_create(c["k2"][i], c["n2"][i], c["b1"][i], c["b2"][i])
        assert l17.p2_eph_verify(e1) and l17.p1_eph_verify(e2, c["b1"][i], c["b2"][i])
        assert not l17.p1_eph_verify(e2, c["b1"][i], c["b2"][i] ^ 1)
        c3 = l17.p2_partial_sig(c["eks"][i], c["c_key"][i], c["x2"][i], c["k2"][i], e1.public_share, c["msg"][i], c["rho"][i], c["r_enc"][i])
        r, s, recid = l17.p1_sign(c["dks"][i], c3, c["k1"][i], e2.public_share)
        assert l17.verify(r, s, c["pub"][i], c["msg"][i])
        assert _ecdsa_ok(r, s, c["pub"][i], c["msg"][i])
        assert not l17.verify(r, Q - s, c["pub"][i], c["msg"][i])          # high s is refused (malleability rule)
        # recovery id: R = (k1 k2) G, parity of y flipped when s was normalised
        Rpt = o.pt_mul(e2.public_share, c["k1"][i])
        s_raw = (pow(c["k1"][i] * c["k2"][i], -1, Q) * (c["msg"][i] + r * c["x1"][i] * c["x2"][i])) % Q
        assert recid == ((Rpt[1] % Q) & 1) ^ (1 if s_raw > Q - s_raw else 0)
    assert l17.p2_partial_sig(c["eks"][0], c["c_key"][0], c["x2"][0], 0, G, 1, 1, 1) is None


def test_zk_pdl_oracle_flow(keyset):
    rng = random.Random(0x9D1)
    c = _l17_case(keyset, rng, 2)
    for i in range(2):
        a, b = rng.randrange(1, Q), rng.randrange(Q * Q)
        Qpt = o.pt_mul(G, c["x1"][i])
        st = l17.pdl_verifier_message1(c["eks"][i], c["c_key"][i], Qpt, a, b, c["r_enc"][i], c["b1"][i] % Q)
        c_hat, q_hat, alpha = l17.pdl_prover_message1(c["dks"][i], st.c_tag, c["b2"][i] % Q)
        assert alpha == a * c["x1"][i] + b
        assert l17.pdl_prover_message2(c["x1"][i], alpha, st.c_tag_tag, a, b, st.blindness)
        assert not l17.pdl_prover_message2(c["x1"][i], alpha, st.c_tag_tag, a, b + 1, st.blindness)
        assert l17.pdl_verifier_finalize(c_hat, q_hat, c["b2"][i] % Q, st.q_tag)
        # a prover whose ciphertext does not hold x1 cannot match Q'
        bad = l17.pdl_verifier_message1(c["eks"][i], o.paillier_encrypt(c["eks"][i], c["x1"][i] + 1, 7), Qpt, a, b, c["r_enc"][i], c["b1"][i] % Q)
        ch2, qh2, _ = l17.pdl_prover_message1(c["dks"][i], bad.c_tag, c["b2"][i] % Q)
        assert not l17.pdl_verifier_finalize(ch2, qh2, c["b2"][i] % Q, bad.q_tag)


def _gg18_case(rng, sessions, parties):
    """Valid GG18 phase-5 inputs: per session a key x, nonce k, R = k^-1 G, additive shares s_i of s = k (m + r x)"""
    U = sessions * parties
    c = dict(parties=parties, sessions=sessions, R=[], y=[], msg=[], s=[], full=[])
    for _ in range(sessions):
        x, k, m = rng.randrange(1, Q), rng.randrange(1, Q), rng.getrandbits(256)
        R = o.pt_mul(G, pow(k, -1, Q))
        s = (m % Q + (R[0] % Q) * x) * k % Q
        parts = [rng.randrange(Q) for _ in range(parties - 1)]
        parts.append((s - sum(parts)) % Q)
        c["R"] += [R] * parties; c["y"] += [o.pt_mul(G, x)] * parties; c["msg"] += [m] * parties; c["s"] += parts; c["full"].append(s)
    for name in ("l", "rho", "hs1", "hs2", "dn"):
        c[name] = [rng.randrange(1, Q) for _ in range(U)]
    for name in ("blind", "blind2"):
        c[name] = [rng.getrandbits(256) for _ in range(U)]
    return c


def _gg18_oracle_run(c):
    P, U = c["parties"], c["parties"] * c["sessions"]
    a5 = [e18.phase5a(c["s"][u], c["l"][u], c["rho"][u], c["R"][u], c["blind"][u], c["hs1"][u], c["hs2"][u], c["dn"][u]) for u in range(U)]
    c5, d5 = [], []
    for u in range(U):
        s0 = u // P * P
        others = [a5[v] for v in range(s0, s0 + P) if v != u]
        c5.append(e18.phase5c(c["msg"][u], c["R"][u], c["y"][u], c["rho"][u], c["l"][u], others, a5[u].V, c["blind2"][u]))
    for u in range(U):
        s0 = u // P * P
        if any(c5[v][0] != e18.OK for v in range(s0, s0 + P)):
            d5.append(None)
            continue
        dec2 = [(c5[v][1][1], c5[v][1][2], c["blind2"][v]) for v in range(s0, s0 + P)]
        d5.append(e18.phase5d(dec2, [c5[v][1][0] for v in range(s0, s0 + P)], [a5[v].B for v in range(s0, s0 + P)]))
    return a5, c5, d5


def test_gg18_phase5_oracle_flow():
    rng = random.Random(0x6618)
    c = _gg18_case(rng, 2, 3)
    a5, c5, d5 = _gg18_oracle_run(c)
    assert all(code == e18.OK for code, _ in c5) and d5 == [e18.OK] * 6
    for sess in range(2):
        code, sig = e18.output_signature(c["R"][3 * sess], c["y"][3 * sess], c["msg"][3 * sess], c["s"][3 * sess:3 * sess + 3])
        assert code == e18.OK and _ecdsa_ok(sig[0], sig[1], c["y"][3 * sess], c["msg"][3 * sess])
    # a wrong share: phase 5c still passes (the proofs are about consistency), phase 5d refuses with InvalidKey
    bad = dict(c); bad["s"] = list(c["s"]); bad["s"][1] = (bad["s"][1] + 1) % Q
    _, c5b, d5b = _gg18_oracle_run(bad)
    assert all(code == e18.OK for code, _ in c5b) and d5b[:3] == [e18.INVALID_KEY] * 3 and d5b[3:] == [e18.OK] * 3
    assert e18.output_signature(bad["R"][0], bad["y"][0], bad["msg"][0], bad["s"][:3])[0] == e18.INVALID_SIG
    # phase 4: commitments and MessageB public keys must match the decommitments
    gam = [rng.randrange(1, Q) for _ in range(3)]
    gg = [o.pt_mul(G, g) for g in gam]
    bl = [rng.getrandbits(256) for _ in range(3)]
    coms = [e18.phase1_broadcast(p, b) for p, b in zip(gg, bl)]
    dinv = rng.randrange(1, Q)
    R = e18.phase4(dinv, gg, list(zip(bl, gg)), coms)
    assert R == o.pt_mul(G, sum(gam) * dinv % Q)
    assert e18.phase4(dinv, [gg[1], gg[1], gg[2]], list(zip(bl, gg)), coms) is None
    assert e18.phase4(dinv, gg, list(zip(bl, gg)), [coms[0] ^ 1] + coms[1:]) is None


# ------------------------------------------------------------------------------------------------ kernels on the host harness
def _pt_limbs(p):
    return np.frombuffer((p[0] | (p[1] << 256)).to_bytes(64, "little"), dtype="<u4")


def _sc_limbs(x, k=8):
    return np.frombuffer(int(x).to_bytes(4 * k, "little"), dtype="<u4")


def _ecddh_row(pf):
    return np.concatenate([_pt_limbs(pf.a1), _pt_limbs(pf.a2), _sc_limbs(pf.z)])


@pytest.fixture(scope="module")
def hh():
    """tests/host_harness: the product's per-element kernels compiled for the CPU (see tests/test_glue_host.py)"""
    import ctypes
    import os
    import subprocess
    import __graft_entry__ as entry
    here = os.path.join(os.path.dirname(os.path.abspath(__file__)), "host_harness")
    so = os.path.join(here, "libglue_host.so")
    srcs = [os.path.join(here, "harness.cpp")] + [os.path.join(entry.CSRC, f) for f in os.listdir(entry.CSRC) if f.endswith((".cuh", ".h"))]
    if not os.path.exists(so) or any(os.path.getmtime(x) > os.path.getmtime(so) for x in srcs):
        subprocess.check_call(["g++", "-O1", "-w", "-I", here, "-I", entry.CSRC, "-shared", "-fPIC", "-o", so, os.path.join(here, "harness.cpp")])
    lib = ctypes.CDLL(so)
    lib.h_init()
    return lib


def _A(vals, k):
    """ints -> (n, k) uint32 limbs"""
    return np.frombuffer(b"".join(int(v).to_bytes(4 * k, "little") for v in vals), dtype="<u4").reshape(len(vals), k).copy()


def _PA(pts):
    return _A([p[0] | (p[1] << 256) for p in pts], 16)


def _I(a):
    return [int.from_bytes(np.ascontiguousarray(r).tobytes(), "little") for r in a]


def _UP(a):
    return [None if v == 0 else (v & ((1 << 256) - 1), v >> 256) for v in _I(a)]


def _call(fn, *args):
    import ctypes
    conv = []
    for a in args:
        if a is None:
            conv.append(ctypes.c_void_p(0))
        elif isinstance(a, np.ndarray):
            conv.append(a.ctypes.data_as(ctypes.c_void_p))
        else:
            conv.append(ctypes.c_int(a))
    fn(*conv)


def test_lindell17_kernels_on_host_harness(hh, keyset):
    rng = random.Random(0x1717)
    n = 6
    c = _l17_case(keyset, rng, n)
    n_tab = _A([keyset[r].dk.p * keyset[r].dk.q for r in range(3)], 64)
    rows = np.asarray(c["rows"], np.uint32)
    # ephemeral keys
    w1 = [l17.eph_create(c["k1"][i], c["n1"][i]) for i in range(n)]
    w2 = [l17.eph_create(c["k2"][i], c["n2"][i], c["b1"][i], c["b2"][i]) for i in range(n)]
    pub, cp, pf = np.zeros((n, 16), np.uint32), np.zeros((n, 16), np.uint32), np.zeros((n, 40), np.uint32)
    c1, c2 = np.zeros((n, 8), np.uint32), np.zeros((n, 8), np.uint32)
    _call(hh.h_l17_eph_create, _A(c["k2"], 8), _A(c["n2"], 8), _A(c["b1"], 8), _A(c["b2"], 8), pub, cp, pf, c1, c2, n)
    assert _UP(pub) == [w.public_share for w in w2] and _UP(cp) == [w.c for w in w2]
    assert np.array_equal(pf, np.stack([_ecddh_row(w.proof) for w in w2]))
    assert _I(c1) == [w.pk_commitment for w in w2] and _I(c2) == [w.zk_pok_commitment for w in w2]
    st = np.full(n, 255, np.uint8)
    _call(hh.h_l17_eph_verify, pub, cp, pf, _A(c["b1"], 8), _A(c["b2"], 8), c1, c2, st, n)
    assert list(st) == [0] * n
    c2b = c2.copy(); c2b[0, 0] ^= 1
    _call(hh.h_l17_eph_verify, pub, cp, pf, _A(c["b1"], 8), _A(c["b2"], 8), c1, c2b, st, n)
    assert list(st) == [11] + [0] * (n - 1)
    cpb = cp.copy(); cpb[[0, 1]] = cp[[1, 0]]
    _call(hh.h_l17_eph_verify, pub, cpb, pf, None, None, None, None, st, n)
    assert list(st) == [10, 10] + [0] * (n - 2)
    # party two: scalar part of PartialSig::compute
    k2 = list(c["k2"]); k2[3] = 0
    v8, lin, st = np.zeros((n, 8), np.uint32), np.zeros((n, 128), np.uint32), np.full(n, 255, np.uint8)
    _call(hh.h_l17_p2_pre, n_tab, rows, _A(c["x2"], 8), _A(k2, 8), _PA([w.public_share for w in w1]), _A(c["msg"], 8), _A(c["rho"], 16), v8, lin, st, n)
    assert list(st) == [4 if i == 3 else 0 for i in range(n)]
    for i in range(n):
        if i == 3:
            continue
        rx = o.pt_mul(w1[i].public_share, k2[i])[0] % Q
        kinv = pow(k2[i], -1, Q)
        assert _I(v8)[i] == kinv * (rx * c["x2"][i] % Q) % Q
        assert _I(lin)[i] == 1 + (c["rho"][i] * Q + kinv * c["msg"][i] % Q) * c["eks"][i].n
    # party one: after the decrypt
    c3 = [l17.p2_partial_sig(c["eks"][i], c["c_key"][i], c["x2"][i], c["k2"][i], w1[i].public_share, c["msg"][i], c["rho"][i], c["r_enc"][i]) for i in range(n)]
    s_tag = [o.paillier_decrypt(c["dks"][i], c3[i]) for i in range(n)]
    r8, s8 = np.zeros((n, 8), np.uint32), np.zeros((n, 8), np.uint32)
    rec = np.zeros(n, np.uint8)
    _call(hh.h_l17_p1_post, _A(s_tag, 64), _A(c["k1"], 8), _PA([w.public_share for w in w2]), r8, s8, rec, st, n)
    want = [l17.p1_sign(c["dks"][i], c3[i], c["k1"][i], w2[i].public_share) for i in range(n)]
    assert list(st) == [0] * n and list(zip(_I(r8), _I(s8), [int(x) for x in rec])) == want
    rr, ss = _I(r8), _I(s8)
    ss[1] = Q - ss[1]; rr[2] = (rr[2] + 1) % Q; ss[4] = 0
    _call(hh.h_l17_verify, _A(rr, 8), _A(ss, 8), _PA(c["pub"]), _A(c["msg"], 8), st, n)
    assert list(st) == [0 if l17.verify(rr[i], ss[i], c["pub"][i], c["msg"][i]) else 9 for i in range(n)] and list(st).count(0) == n - 3


def test_zk_pdl_kernels_on_host_harness(hh, keyset):
    rng = random.Random(0x2D1)
    n = 6
    c = _l17_case(keyset, rng, n)
    n_tab = _A([keyset[r].dk.p * keyset[r].dk.q for r in range(3)], 64)
    rows = np.asarray(c["rows"], np.uint32)
    a = [rng.randrange(1, Q) for _ in range(n)]
    a[0] = 1; a[1] = (1 << 255) | 5; a[2] = 0xFFFFFFFF
    b = [rng.randrange(Q * Q) for _ in range(n)]
    b[3] = 0
    bl_v, bl_p = [x % Q for x in c["b1"]], [x % Q for x in c["b2"]]
    Qs = [o.pt_mul(G, x) for x in c["x1"]]
    want = [l17.pdl_verifier_message1(c["eks"][i], c["c_key"][i], Qs[i], a[i], b[i], c["r_enc"][i], bl_v[i]) for i in range(n)]
    lin, ctt, qt, st = np.zeros((n, 128), np.uint32), np.zeros((n, 8), np.uint32), np.zeros((n, 16), np.uint32), np.full(n, 255, np.uint8)
    _call(hh.h_zkpdl_v1_pre, n_tab, rows, _PA(Qs), _A(a, 8), _A(b, 16), _A(bl_v, 8), lin, ctt, qt, st, n)
    assert list(st) == [0] * n and _I(ctt) == [w.c_tag_tag for w in want] and _UP(qt) == [w.q_tag for w in want]
    assert _I(lin) == [1 + b[i] * c["eks"][i].n for i in range(n)]
    alpha = [a[i] * c["x1"][i] + b[i] for i in range(n)]
    ch, qh = np.zeros((n, 8), np.uint32), np.zeros((n, 16), np.uint32)
    _call(hh.h_zkpdl_p1_post, _A(alpha, 64), _A(bl_p, 8), ch, qh, st, n)
    want_p = [l17.pdl_prover_message1(c["dks"][i], want[i].c_tag, bl_p[i]) for i in range(n)]
    assert list(st) == [0] * n and list(zip(_I(ch), _UP(qh))) == [(w[0], w[1]) for w in want_p] and [w[2] for w in want_p] == alpha
    _call(hh.h_zkpdl_p2, _A(c["x1"], 8), _A(alpha, 64), ctt, _A(a, 8), _A(b, 16), _A(bl_v, 8), st, n)
    assert list(st) == [0] * n
    b_bad = list(b); b_bad[4] += 1
    _call(hh.h_zkpdl_p2, _A(c["x1"], 8), _A(alpha, 64), ctt, _A(a, 8), _A(b_bad, 16), _A(bl_v, 8), st, n)
    assert list(st) == [6 if i == 4 else 0 for i in range(n)]
    _call(hh.h_zkpdl_finalize, ch, qh, _A(bl_p, 8), qt, st, n)
    assert list(st) == [0] * n
    qtb = qt.copy(); qtb[[0, 1]] = qt[[1, 0]]
    _call(hh.h_zkpdl_finalize, ch, qh, _A(bl_p, 8), qtb, st, n)
    assert list(st) == [6, 6] + [0] * (n - 2)


def test_gg18_kernels_on_host_harness(hh):
    rng = random.Random(0x1818)
    for parties, sessions in ((2, 2), (3, 2)):
        c = _gg18_case(rng, sessions, parties)
        U = parties * sessions
        c["s"][parties] = (c["s"][parties] + 1) % Q
        a5, c5, d5 = _gg18_oracle_run(c)
        com, vab, heg, dlog = np.zeros((U, 8), np.uint32), np.zeros((U, 48), np.uint32), np.zeros((U, 48), np.uint32), np.zeros((U, 40), np.uint32)
        st = np.full(U, 255, np.uint8)
        _call(hh.h_gg18_phase5a, _PA(c["R"]), _A(c["s"], 8), _A(c["l"], 8), _A(c["rho"], 8), _A(c["blind"], 8), _A(c["hs1"], 8), _A(c["hs2"], 8), _A(c["dn"], 8),
              com, vab, heg, dlog, st, U)
        assert list(st) == [0] * U
        for u in range(U):
            w = a5[u]
            assert _I(com)[u] == w.com
            assert np.array_equal(vab[u], np.concatenate([_pt_limbs(w.V), _pt_limbs(w.A), _pt_limbs(w.B)]))
            assert np.array_equal(heg[u], np.concatenate([_pt_limbs(w.heg.T), _pt_limbs(w.heg.A3), _sc_limbs(w.heg.z1), _sc_limbs(w.heg.z2)]))
            assert np.array_equal(dlog[u], np.concatenate([_pt_limbs(w.dlog.pk), _pt_limbs(w.dlog.pk_t_rand_commitment), _sc_limbs(w.dlog.challenge_response)]))
        com2, ut = np.zeros((U, 8), np.uint32), np.zeros((U, 32), np.uint32)
        args5c = lambda cm, hg, dl: (parties, _PA(c["R"]), _PA(c["y"]), _A(c["msg"], 8), _A(c["rho"], 8), _A(c["l"], 8), _A(c["blind2"], 8), cm, vab, _A(c["blind"], 8),
                                     hg, dl, com2, ut, st, U)
        _call(hh.h_gg18_phase5c, *args5c(com, heg, dlog))
        assert list(st) == [code for code, _ in c5] == [0] * U
        for u in range(U):
            assert _I(com2)[u] == c5[u][1][0] and np.array_equal(ut[u], np.concatenate([_pt_limbs(c5[u][1][1]), _pt_limbs(c5[u][1][2])]))
        good_com2, good_ut = com2.copy(), ut.copy()
        for field in ("com", "heg", "dlog"):
            cm, hg, dl = com.copy(), heg.copy(), dlog.copy()
            if field == "com":
                cm[0, 0] ^= 1
            elif field == "heg":
                hg[0] = heg[1]
            else:
                dl[0, 32] ^= 1                                             # a VALID foreign DLogProof would pass: the reference never ties pk to A_i
            _call(hh.h_gg18_phase5c, *args5c(cm, hg, dl))
            assert list(st[:parties]) == [0] + [11] * (parties - 1) and list(st[parties:]) == [0] * (U - parties), field
        _call(hh.h_gg18_phase5d, parties, good_ut, _A(c["blind2"], 8), good_com2, vab, st, U)
        assert list(st) == d5 and list(st[:parties]) == [0] * parties and list(st[parties:2 * parties]) == [2] * parties
        bad_com2 = good_com2.copy(); bad_com2[0, 0] ^= 1
        _call(hh.h_gg18_phase5d, parties, good_ut, _A(c["blind2"], 8), bad_com2, vab, st, U)
        assert list(st[:parties]) == [11] * parties
        sr, ss, rec = np.zeros((U, 8), np.uint32), np.zeros((U, 8), np.uint32), np.zeros(U, np.uint8)
        _call(hh.h_gg18_output, parties, _PA(c["R"]), _PA(c["y"]), _A(c["msg"], 8), _A(c["s"], 8), sr, ss, rec, st, U)
        for sess in range(sessions):
            u0 = sess * parties
            code, sig = e18.output_signature(c["R"][u0], c["y"][u0], c["msg"][u0], c["s"][u0:u0 + parties])
            assert all(int(st[u]) == code for u in range(u0, u0 + parties))
            if code == 0:
                assert all((_I(sr)[u], _I(ss)[u], int(rec[u])) == sig for u in range(u0, u0 + parties))
        k_i, sg = [rng.randrange(1, Q) for _ in range(U)], [rng.randrange(1, Q) for _ in range(U)]
        s_i = np.zeros((U, 8), np.uint32)
        _call(hh.h_gg18_local_sig, _A(c["msg"], 8), _PA(c["R"]), _A(k_i, 8), _A(sg, 8), s_i, U)
        assert _I(s_i) == [e18.phase5_local_sig(k_i[u], c["msg"][u], c["R"][u], sg[u]) for u in range(U)]
        gam = [rng.randrange(1, Q) for _ in range(U)]
        gg = [o.pt_mul(G, g) for g in gam]
        bl = [rng.getrandbits(256) for _ in range(U)]
        coms = [e18.phase1_broadcast(p, b) for p, b in zip(gg, bl)]
        dinv = [rng.randrange(1, Q) for _ in range(U)]
        pks = [[gg[u // parties * parties + j] for j in range(parties)] for u in range(U)]
        pks[1][0] = gg[1]
        R4 = np.zeros((U, 16), np.uint32)
        _call(hh.h_gg18_phase4, parties, _A(dinv, 8), _PA([p for row in pks for p in row]), _PA(gg), _A(bl, 8), _A(coms, 8), R4, st, U)
        for u in range(U):
            s0 = u // parties * parties
            want = e18.phase4(dinv[u], pks[u], [(bl[v], gg[v]) for v in range(s0, s0 + parties)], coms[s0:s0 + parties])
            assert (int(st[u]) == 0) == (want is not None) and (want is None or _UP(R4)[u] == want)
        assert int(st[1]) == 2 and int(st[0]) == 0


# ------------------------------------------------------------------------------------------------ GPU parity
@pytest.mark.gpu
def test_lindell17_on_gpu_matches_oracle(engine, pkg, keyset):
    from mpecdsa_b200 import gg20, lindell17 as L
    rng = random.Random(0x1717)
    n = 12
    c = _l17_case(keyset, rng, n)
    ks = gg20.KeySets(engine, [keyset])
    n_list = [keyset[r].dk.p * keyset[r].dk.q for r in range(3)]
    # key generation messages
    com1, com2, pk, proof = L.p1_keygen_first(engine, c["x1"], c["n1"], c["b1"], c["b2"])
    want = [l17.p1_keygen_first(c["x1"][i], c["n1"][i], c["b1"][i], c["b2"][i]) for i in range(n)]
    assert com1 == [w.pk_commitment for w in want] and com2 == [w.zk_pok_commitment for w in want] and pk == [w.public_share for w in want]
    assert list(L.p2_keygen_verify(engine, com1, com2, pk, proof, c["b1"], c["b2"])) == [0] * n
    assert list(L.p2_keygen_verify(engine, com1, [com2[0] ^ 1] + com2[1:], pk, proof, c["b1"], c["b2"])) == [pkg.ST_COMMITMENT] + [0] * (n - 1)
    # ephemeral keys, both parties
    e1 = L.eph_create(engine, c["k1"], c["n1"])
    e2 = L.eph_create(engine, c["k2"], c["n2"], c["b1"], c["b2"])
    w1 = [l17.eph_create(c["k1"][i], c["n1"][i]) for i in range(n)]
    w2 = [l17.eph_create(c["k2"][i], c["n2"][i], c["b1"][i], c["b2"][i]) for i in range(n)]
    for got, want in ((e1, w1), (e2, w2)):
        assert got["public_share"] == [w.public_share for w in want] and got["c"] == [w.c for w in want]
        assert np.array_equal(got["proof"], np.stack([_ecddh_row(w.proof) for w in want]))
    assert e1["pk_commitment"] is None
    assert e2["pk_commitment"] == [w.pk_commitment for w in w2] and e2["zk_pok_commitment"] == [w.zk_pok_commitment for w in w2]
    assert list(L.eph_verify(engine, e1["public_share"], e1["c"], e1["proof"])) == [0] * n
    assert list(L.eph_verify(engine, e2["public_share"], e2["c"], e2["proof"], c["b1"], c["b2"], e2["pk_commitment"], e2["zk_pok_commitment"])) == [0] * n
    bad_blind = [c["b2"][0] ^ 1] + c["b2"][1:]
    assert list(L.eph_verify(engine, e2["public_share"], e2["c"], e2["proof"], c["b1"], bad_blind, e2["pk_commitment"], e2["zk_pok_commitment"])) == [pkg.ST_COMMITMENT] + [0] * (n - 1)
    swapped = [e1["c"][1], e1["c"][0]] + e1["c"][2:]
    assert list(L.eph_verify(engine, e1["public_share"], swapped, e1["proof"])) == [pkg.ST_PROOF] * 2 + [0] * (n - 2)
    # party two's partial signature and party one's signature
    k2 = list(c["k2"]); k2[3] = 0
    c3, st = L.p2_partial_sig(engine, n_list, c["rows"], c["c_key"], c["x2"], k2, e1["public_share"], c["msg"], c["rho"], c["r_enc"])
    want_c3 = [l17.p2_partial_sig(c["eks"][i], c["c_key"][i], c["x2"][i], k2[i], w1[i].public_share, c["msg"][i], c["rho"][i], c["r_enc"][i]) for i in range(n)]
    assert list(st) == [pkg.ST_NOT_INVERTIBLE if i == 3 else 0 for i in range(n)]
    assert all(c3[i] == want_c3[i] for i in range(n) if i != 3)
    c3[3] = want_c3[3] = l17.p2_partial_sig(c["eks"][3], c["c_key"][3], c["x2"][3], c["k2"][3], w1[3].public_share, c["msg"][3], c["rho"][3], c["r_enc"][3])
    r, s, rec, st = L.p1_sign(engine, ks, c["rows"], c3, c["k1"], e2["public_share"])
    want = [l17.p1_sign(c["dks"][i], c3[i], c["k1"][i], w2[i].public_share) for i in range(n)]
    assert list(st) == [0] * n and list(zip(r, s, [int(x) for x in rec])) == want
    assert all(_ecdsa_ok(r[i], s[i], c["pub"][i], c["msg"][i]) for i in range(n))
    # verify, with the reference's corner cases: high s, r given as x >= q is impossible here so r + 1 instead, s = 0
    rr, ss = list(r) * 1, list(s) * 1
    ss[1] = Q - ss[1]; rr[2] = (rr[2] + 1) % Q; ss[4] = 0
    got = list(L.verify(engine, rr, ss, c["pub"], c["msg"]))
    assert got == [0 if l17.verify(rr[i], ss[i], c["pub"][i], c["msg"][i]) else pkg.ST_INVALID_SIG for i in range(n)]
    assert got[1] == got[2] == got[4] == pkg.ST_INVALID_SIG and got.count(0) == n - 3
    ks.free()


@pytest.mark.gpu
def test_zk_pdl_on_gpu_matches_oracle(engine, pkg, keyset):
    from mpecdsa_b200 import gg20, lindell17 as L
    rng = random.Random(0x2D1)
    n = 9
    c = _l17_case(keyset, rng, n)
    ks = gg20.KeySets(engine, [keyset])
    n_list = [keyset[r].dk.p * keyset[r].dk.q for r in range(3)]
    a = [rng.randrange(1, Q) for _ in range(n)]
    a[0] = 1; a[1] = (1 << 255) | 5; a[2] = 0xFFFFFFFF                   # bit_length(a) on and off limb boundaries
    b = [rng.randrange(Q * Q) for _ in range(n)]
    bl_v = [x % Q for x in c["b1"]]
    bl_p = [x % Q for x in c["b2"]]
    Qs = [o.pt_mul(G, x) for x in c["x1"]]
    ct, ctt, qt, st = L.pdl_verifier_message1(engine, n_list, c["rows"], c["c_key"], Qs, a, b, c["r_enc"], bl_v)
    want = [l17.pdl_verifier_message1(c["eks"][i], c["c_key"][i], Qs[i], a[i], b[i], c["r_enc"][i], bl_v[i]) for i in range(n)]
    assert list(st) == [0] * n
    assert ct == [w.c_tag for w in want] and ctt == [w.c_tag_tag for w in want] and qt == [w.q_tag for w in want]
    ch, qh, al, st = L.pdl_prover_message1(engine, ks, c["rows"], ct, bl_p)
    want_p = [l17.pdl_prover_message1(c["dks"][i], ct[i], bl_p[i]) for i in range(n)]
    assert list(st) == [0] * n and list(zip(ch, qh, al)) == want_p
    b_bad = list(b); b_bad[4] += 1
    assert list(L.pdl_prover_message2(engine, c["x1"], al, ctt, a, b, bl_v)) == [0] * n
    assert list(L.pdl_prover_message2(engine, c["x1"], al, ctt, a, b_bad, bl_v)) == [pkg.ST_PDL_VERIFY if i == 4 else 0 for i in range(n)]
    assert list(L.pdl_verifier_finalize(engine, ch, qh, bl_p, qt)) == [0] * n
    qt_bad = [qt[1], qt[0]] + qt[2:]
    assert list(L.pdl_verifier_finalize(engine, ch, qh, bl_p, qt_bad)) == [pkg.ST_PDL_VERIFY] * 2 + [0] * (n - 2)
    ks.free()


@pytest.mark.gpu
def test_gg18_phases_on_gpu_match_oracle(engine, pkg):
    from mpecdsa_b200 import gg18
    rng = random.Random(0x1818)
    for parties, sessions in ((2, 5), (3, 4), (5, 2)):
        c = _gg18_case(rng, sessions, parties)
        U = parties * sessions
        c["s"][parties] = (c["s"][parties] + 1) % Q                      # second session: one wrong share
        a5, c5, d5 = _gg18_oracle_run(c)
        got = gg18.phase5a(engine, c["R"], c["s"], c["l"], c["rho"], c["blind"], c["hs1"], c["hs2"], c["dn"])
        assert list(got["status"]) == [0] * U
        for u in range(U):
            w = a5[u]
            assert int.from_bytes(got["com"][u].tobytes(), "little") == w.com
            assert np.array_equal(got["decom"][u], np.concatenate([_pt_limbs(w.V), _pt_limbs(w.A), _pt_limbs(w.B)]))
            assert np.array_equal(got["heg"][u], np.concatenate([_pt_limbs(w.heg.T), _pt_limbs(w.heg.A3), _sc_limbs(w.heg.z1), _sc_limbs(w.heg.z2)]))
            assert np.array_equal(got["dlog"][u], np.concatenate([_pt_limbs(w.dlog.pk), _pt_limbs(w.dlog.pk_t_rand_commitment), _sc_limbs(w.dlog.challenge_response)]))
        g5c = gg18.phase5c(engine, parties, c["R"], c["y"], c["msg"], c["rho"], c["l"], c["blind2"], got["com"], got["decom"], c["blind"], got["heg"], got["dlog"])
        assert list(g5c["status"]) == [code for code, _ in c5] == [0] * U
        for u in range(U):
            com2, ui, ti = c5[u][1]
            assert int.from_bytes(g5c["com2"][u].tobytes(), "little") == com2
            assert np.array_equal(g5c["decom2"][u], np.concatenate([_pt_limbs(ui), _pt_limbs(ti)]))
        g5d = gg18.phase5d(engine, parties, g5c["decom2"], c["blind2"], g5c["com2"], got["decom"])
        assert list(g5d) == d5
        assert list(g5d[parties:2 * parties]) == [pkg.ST_INVALID_KEY] * parties and list(g5d[:parties]) == [0] * parties
        r, s, rec, st = gg18.output_signature(engine, parties, c["R"], c["y"], c["msg"], c["s"])
        for sess in range(sessions):
            u0 = sess * parties
            code, sig = e18.output_signature(c["R"][u0], c["y"][u0], c["msg"][u0], c["s"][u0:u0 + parties])
            assert all(int(st[u]) == code for u in range(u0, u0 + parties))
            if code == 0:
                assert all((r[u], s[u], int(rec[u])) == sig for u in range(u0, u0 + parties))
                assert _ecdsa_ok(r[u0], s[u0], c["y"][u0], c["msg"][u0])
        assert int(st[parties]) == pkg.ST_INVALID_SIG
        # tampering with the phase-5a messages: a flipped commitment, a foreign ElGamal proof, a corrupted DLog proof
        for field, code in (("com", pkg.ST_COMMITMENT), ("heg", pkg.ST_COMMITMENT), ("dlog", pkg.ST_COMMITMENT)):
            t = {k: v.copy() for k, v in got.items()}
            if field == "com":
                t["com"][0, 0] ^= 1
            elif field == "heg":
                t["heg"][0] = got["heg"][1]
            else:
                t["dlog"][0, 32] ^= 1                                      # a VALID foreign DLogProof would pass: the reference never ties pk to A_i
            st_t = gg18.phase5c(engine, parties, c["R"], c["y"], c["msg"], c["rho"], c["l"], c["blind2"], t["com"], t["decom"], c["blind"], t["heg"], t["dlog"])["status"]
            # element 0's message is checked by the OTHER signers of its session only
            assert list(st_t[:parties]) == [0] + [code] * (parties - 1) and list(st_t[parties:]) == [0] * (U - parties), field
        # local signature share
        k_i, sig_i = [rng.randrange(1, Q) for _ in range(U)], [rng.randrange(1, Q) for _ in range(U)]
        assert gg18.local_sig(engine, c["msg"], c["R"], k_i, sig_i) == [e18.phase5_local_sig(k_i[u], c["msg"][u], c["R"][u], sig_i[u]) for u in range(U)]
        # phase 4
        gam = [rng.randrange(1, Q) for _ in range(U)]
        gg = [o.pt_mul(G, g) for g in gam]
        bl = [rng.getrandbits(256) for _ in range(U)]
        coms = [e18.phase1_broadcast(p, b) for p, b in zip(gg, bl)]
        dinv = [rng.randrange(1, Q) for _ in range(U)]
        pks = [[gg[u // parties * parties + j] for j in range(parties)] for u in range(U)]
        pks[1][0] = gg[1]                                                  # element 1 holds a wrong public key for signer 0
        R4, st4 = gg18.phase4(engine, parties, dinv, pks, gg, bl, coms)
        for u in range(U):
            s0 = u // parties * parties
            want = e18.phase4(dinv[u], pks[u], [(bl[v], gg[v]) for v in range(s0, s0 + parties)], coms[s0:s0 + parties])
            assert (int(st4[u]) == 0) == (want is not None) and (want is None or R4[u] == want)
        assert int(st4[1]) == pkg.ST_INVALID_KEY and int(st4[0]) == 0


@pytest.mark.gpu
def test_gg18_whole_signing_on_gpu(engine, pkg, keyset):
    """gg_2018/test.rs `sign` as batch calls: two- and three-signer sessions over the (t=1, n=3) key set, phases 1-5; the signature
    verifies under OpenSSL and equals k^-1 (m + r x) computed from the opened secrets; a wrong share is caught in phase 5d"""
    from mpecdsa_b200 import gg18, gg20
    ks = gg20.KeySets(engine, [keyset])
    y = keyset[0].y_sum_s
    rng = random.Random(0x6718)
    for signers_list in ([[0, 1], [0, 2], [1, 2], [2, 0]], [[0, 1, 2], [2, 1, 0]]):
        parties = len(signers_list[0])
        U = parties * len(signers_list)
        P1 = parties - 1
        rows = [p for s in signers_list for p in s]
        w = [o.lagrange_at_zero(p, s) * keyset[p].x_i % Q for s in signers_list for p in s]
        msg = [m for s in signers_list for m in [rng.getrandbits(256)] * parties]
        sc = lambda n_: [rng.randrange(1, Q) for _ in range(n_)]
        nmod = lambda elems: [rng.randrange(1, keyset[rows[u]].dk.p * keyset[rows[u]].dk.q) for u in elems]
        alice = [u for u in range(U) for _ in range(P1)]
        rnd = dict(k=sc(U), gamma=sc(U), blind=[rng.getrandbits(256) for _ in range(U)], r_a=nmod(range(U)), l=sc(U), rho=sc(U),
                   blind5=[rng.getrandbits(256) for _ in range(U)], blind5c=[rng.getrandbits(256) for _ in range(U)], heg_s1=sc(U), heg_s2=sc(U), dlog_nonce=sc(U),
                   r_b_gamma=nmod(alice), r_b_w=nmod(alice), nb_gamma=sc(U * P1), nbt_gamma=sc(U * P1), nb_w=sc(U * P1), nbt_w=sc(U * P1),
                   beta_tag_gamma=[rng.randrange(keyset[rows[u]].dk.p * keyset[rows[u]].dk.q >> 1) for u in alice],
                   beta_tag_w=[rng.randrange(keyset[rows[u]].dk.p * keyset[rows[u]].dk.q >> 1) for u in alice])
        out = gg18.sign_batch(engine, ks, parties, rows, w, [y] * U, msg, rnd)
        assert list(out["status"]) == [0] * U
        x = sum(o.lagrange_at_zero(p, [0, 1]) * keyset[p].x_i for p in (0, 1)) % Q
        assert o.pt_mul(G, x) == y
        for si in range(len(signers_list)):
            u0 = si * parties
            kk = sum(rnd["k"][u0:u0 + parties]) % Q
            gam = sum(rnd["gamma"][u0:u0 + parties]) % Q
            R = o.pt_mul(G, pow(kk, -1, Q))                         # R = (k gamma)^-1 * gamma G
            assert all(out["R"][u] == R for u in range(u0, u0 + parties)) and gam != 0
            s = kk * (msg[u0] + (R[0] % Q) * x) % Q
            s = min(s, Q - s)
            assert all((out["r"][u], out["s"][u]) == (R[0] % Q, s) for u in range(u0, u0 + parties))
            assert _ecdsa_ok(out["r"][u0], out["s"][u0], y, msg[u0])
        bad_w = list(w); bad_w[0] = (bad_w[0] + 1) % Q
        out = gg18.sign_batch(engine, ks, parties, rows, bad_w, [y] * U, msg, rnd)
        assert list(out["status"][:parties]) == [pkg.ST_INVALID_KEY] * parties and list(out["status"][parties:]) == [0] * (U - parties)
    ks.free()


@pytest.mark.gpu
def test_other_protocol_entry_points_reject_bad_arguments(engine, pkg):
    """API-level errors never reach a kernel: empty batches return 0, NULL buffers and out-of-range signer counts return TECDSA_E_ARG"""
    import ctypes
    from mpecdsa_b200 import gg18, lindell17
    gg18._bind(engine.lib); lindell17._bind(engine.lib)
    lib, ctx = engine.lib, engine._ctx
    z8, z16, z40, z48 = (np.zeros((1, k), np.uint32) for k in (8, 16, 40, 48))
    st = np.zeros(1, np.uint8)
    P = lambda a: a.ctypes.data
    assert lib.tecdsa_l17_verify_batch(ctx, P(z8), P(z8), P(z16), P(z8), P(st), 0, pkg.HOST) == 0
    assert lib.tecdsa_l17_verify_batch(ctx, None, P(z8), P(z16), P(z8), P(st), 1, pkg.HOST) == -1
    assert lib.tecdsa_l17_eph_create_batch(ctx, P(z8), P(z8), P(z8), None, P(z16), P(z16), P(z40), None, None, 1, pkg.HOST) == -1     # half of the commitment buffers
    assert b"come together" in lib.tecdsa_last_error()
    assert lib.tecdsa_gg18_phase5d_batch(ctx, 1, P(z16), P(z8), P(z8), P(z48), P(st), 1, pkg.HOST) == -1                               # one signer is not a session
    assert lib.tecdsa_gg18_phase5d_batch(ctx, 65, P(z16), P(z8), P(z8), P(z48), P(st), 1, pkg.HOST) == -1
    assert lib.tecdsa_gg18_phase5d_batch(ctx, 2, P(z16), P(z8), P(z8), P(z48), P(st), 0, pkg.HOST) == 0
    assert lib.tecdsa_zkpdl_verifier_finalize_batch(ctx, P(z8), P(z16), P(z8), None, P(st), 1, pkg.HOST) == -1
    # points that are not on the curve are a per-element status, not an API error
    bad = np.ones((2, 16), np.uint32)
    st2 = np.full(2, 255, np.uint8)
    assert lib.tecdsa_l17_verify_batch(ctx, P(np.ones((2, 8), np.uint32)), P(np.ones((2, 8), np.uint32)), P(bad), P(np.ones((2, 8), np.uint32)), P(st2), 2, pkg.HOST) == 0
    assert list(st2) == [pkg.ST_INVALID_SIG] * 2


@pytest.mark.gpu
def test_lindell17_wrappers_reject_malformed_peer_values_per_element(engine, pkg, keyset):
    """Values a peer controls (ciphertexts, points, signature halves, decommitments) that do not fit their ABI slot reject that ONE
    element with the status the reference's deserialisation / comparison would lead to; the batch goes through"""
    from mpecdsa_b200 import gg20, lindell17 as L
    rng = random.Random(0x5C12)
    n = 4
    c = _l17_case(keyset, rng, n)
    ks = gg20.KeySets(engine, [keyset])
    n_list = [keyset[r].dk.p * keyset[r].dk.q for r in range(3)]
    e1 = L.eph_create(engine, c["k1"], c["n1"])
    e2 = L.eph_create(engine, c["k2"], c["n2"], c["b1"], c["b2"])
    wide_pt = (1 << 256, 5)
    pubs = list(e1["public_share"]); pubs[1] = wide_pt
    assert list(L.eph_verify(engine, pubs, e1["c"], e1["proof"])) == [0, pkg.ST_PROOF, 0, 0]
    c_key = list(c["c_key"]); c_key[2] = 1 << 4096
    c3, st = L.p2_partial_sig(engine, n_list, c["rows"], c_key, c["x2"], c["k2"], pubs, c["msg"], c["rho"], c["r_enc"])
    assert list(st) == [0, pkg.ST_INVALID_KEY, pkg.ST_INVALID_KEY, 0]
    c3[1] = c3[2] = -5
    r, s, rec, st = L.p1_sign(engine, ks, c["rows"], c3, c["k1"], e2["public_share"])
    assert list(st) == [0, pkg.ST_INVALID_KEY, pkg.ST_INVALID_KEY, 0]
    r[3] = 1 << 300
    assert list(L.verify(engine, r, s, c["pub"], c["msg"])) == [0, pkg.ST_INVALID_SIG, pkg.ST_INVALID_SIG, pkg.ST_INVALID_SIG]
    ks.free()


@pytest.mark.gpu
def test_lindell17_full_key_gen_on_gpu(engine, pkg, keyset):
    """lindell_2017/test.rs `test_full_key_gen` as batch calls: commitments + DLog proof, Paillier-encrypted share, NiCorrectKeyProof,
    PDL-with-slack proof against a freshly generated (N~, h1, h2) with its CompositeDLogProof — every proof checked by the engine's
    verifier AND by the oracle's, and a wrong Q1 / foreign statement rejected"""
    import dataclasses
    from mpecdsa_b200 import gg20, lindell17 as L
    from oracle import keygen_oracle as kg
    from tests.test_keygen_oracle import _setup
    rng = random.Random(0x17F6)
    n = 2
    setups = [_setup(rng, bits=1024) for _ in range(n)]
    params = L.generate_h1_h2_n_tilde(engine, setups)
    for (nt, h1, h2, xhi), (p_t, q_t, h1_in, xhi_in) in zip(params, setups):
        assert nt == p_t * q_t and h2 == pow(pow(h1, -1, nt), xhi, nt) and (h1, xhi) == (h1_in, xhi_in)         # party_one.rs:594-607
    # key rows 0 and 1 of a key set carry party one's Paillier keys and the fresh statements
    parties = []
    for i in range(3):
        lk = keyset[i]
        if i < n:
            st = o.DLogStatement(params[i][0], params[i][1], params[i][2])
            vec = list(lk.h1_h2_n_tilde_vec); vec[lk.i - 1] = st
            lk = dataclasses.replace(lk, h1_h2_n_tilde_vec=vec)
        parties.append(lk)
    ks = gg20.KeySets(engine, [parties])
    x1 = [rng.randrange(1, Q // 3) for _ in range(n)]
    nonce, b1, b2 = [rng.randrange(1, Q) for _ in range(n)], [rng.getrandbits(256) for _ in range(n)], [rng.getrandbits(256) for _ in range(n)]
    com1, com2, pk, proof = L.p1_keygen_first(engine, x1, nonce, b1, b2)
    assert list(L.p2_keygen_verify(engine, com1, com2, pk, proof, b1, b2)) == [0] * n
    p_q = [(keyset[i].dk.p, keyset[i].dk.q) for i in range(n)]
    n_list = [p * q for p, q in p_q]
    stm = [(prm[0], prm[1], prm[2]) for prm in params]
    r_key = [rng.randrange(1, nn) for nn in n_list]
    pdl_rand = ([rng.randrange(Q ** 3) for _ in range(n)], [rng.randrange(1, nn) for nn in n_list], [rng.randrange(Q * s[0]) for s in stm],
                [rng.randrange(Q ** 3 * s[0]) for s in stm])
    msg = L.p1_paillier_and_proofs(engine, ks, list(range(n)), list(range(n)), stm, [prm[3] for prm in params], x1, r_key, pdl_rand,
                                   [rng.getrandbits(500) for _ in range(n)], p_q)
    assert msg["Q"] == pk and msg["encrypted_share"] == [o.paillier_encrypt(o.EncryptionKey(nn, nn * nn), x, r) for nn, x, r in zip(n_list, x1, r_key)]
    assert list(L.p2_verify_paillier_and_proofs(engine, ks, list(range(n)), list(range(n)), stm, n_list, msg, pk)) == [0] * n
    # the oracle's verifiers accept the engine's proofs too
    for i in range(n):
        ek = o.EncryptionKey(n_list[i], n_list[i] ** 2)
        st = o.DLogStatement(*stm[i])
        assert kg.correct_key_verify(msg["correct_key_proof"][i], ek)
        x_, y_ = msg["composite_dlog_proof"][i]
        assert kg.composite_dlog_verify(kg.CompositeDLogProof(x_, y_), st)
        pd = {k_: v[i] for k_, v in msg["pdl"].items()}
        pf = o.PDLwSlackProof(pd["z"], pd["u1"], pd["u2"], pd["u3"], pd["s1"], pd["s2"], pd["s3"])
        assert o.pdl_verify(pf, msg["encrypted_share"][i], ek, pk[i], G, st.g, st.ni, st.N)
    # party two holds a different Q1 for element 0; element 1 is checked against the other element's statement
    assert list(L.p2_verify_paillier_and_proofs(engine, ks, list(range(n)), list(range(n)), stm, n_list, msg, [pk[1], pk[1]])) == [pkg.ST_PDL_VERIFY, 0]
    assert list(L.p2_verify_paillier_and_proofs(engine, ks, list(range(n)), [1, 1], [stm[1], stm[1]], n_list, msg, pk)) == [pkg.ST_PDL_VERIFY, 0]
    ks.free()


@pytest.mark.gpu
def test_gg18_key_generation_then_signing_on_gpu(engine, pkg, keyset):
    """gg_2018/test.rs `keygen_t_n_parties` + `sign` as batch calls: two groups of three parties generate (t = 1, n = 3) keys over the
    fixture Paillier keys, the shares are Shamir-consistent with the group key, and two of the three sign with them; a tampered share
    stops its receiver with InvalidSS"""
    from mpecdsa_b200 import gg18, gg20
    from oracle import keygen_oracle as kg
    rng = random.Random(0x18C9)
    t, n, groups = 1, 3, 2
    E = n * groups
    u = [rng.randrange(1, Q) for _ in range(E)]
    polys = [[u[e]] + [rng.randrange(1, Q) for _ in range(t)] for e in range(E)]
    p_q = [(keyset[e % n].dk.p, keyset[e % n].dk.q) for e in range(E)]
    blind = [rng.getrandbits(256) for _ in range(E)]
    nonce = [rng.randrange(1, Q) for _ in range(E)]
    out = gg18.keygen_batch(engine, t, n, u, p_q, blind, polys, nonce)
    assert list(out["status"]) == [0] * E
    for g in range(groups):
        ys = o.pt_mul(G, sum(u[g * n:(g + 1) * n]) % Q)
        assert all(out["y"][e] == ys for e in range(g * n, (g + 1) * n))
        for e in range(g * n, (g + 1) * n):
            vss, sh = kg.vss_share(t, n, polys[e][0], polys[e][1:])
            assert out["shares"][e] == sh and out["commitments"][e] == vss.commitments
            assert out["x_i"][e] == sum(kg.vss_share(t, n, polys[s][0], polys[s][1:])[1][e % n] for s in range(g * n, (g + 1) * n)) % Q
            assert kg.correct_key_verify(out["correct_key_proof"][e], o.EncryptionKey(p_q[e][0] * p_q[e][1], (p_q[e][0] * p_q[e][1]) ** 2))
        for pair in ([0, 1], [0, 2], [1, 2]):                             # any two shares interpolate the group secret
            lam = [o.lagrange_at_zero(i, pair) for i in pair]
            assert o.pt_mul(G, sum(l * out["x_i"][g * n + i] for l, i in zip(lam, pair)) % Q) == ys
    # sign with parties (0, 2) of group 0 and (1, 2) of group 1 using the freshly generated shares (the Paillier rows are the fixture's)
    ks = gg20.KeySets(engine, [keyset])
    signers = [[0, 2], [1, 2]]
    rows = [p for s in signers for p in s]
    w = [o.lagrange_at_zero(p, s) * out["x_i"][g * n + p] % Q for g, s in enumerate(signers) for p in s]
    ysig = [out["y"][g * n] for g, s in enumerate(signers) for _ in s]
    msg = [m for _ in signers for m in [rng.getrandbits(256)] * 2]
    U, P1 = 4, 1
    sc = lambda m_: [rng.randrange(1, Q) for _ in range(m_)]
    nm = lambda elems: [rng.randrange(1, (keyset[rows[e]].dk.p * keyset[rows[e]].dk.q) >> 1) for e in elems]
    alice = list(range(U))
    rnd = dict(k=sc(U), gamma=sc(U), blind=sc(U), r_a=nm(range(U)), l=sc(U), rho=sc(U), blind5=sc(U), blind5c=sc(U), heg_s1=sc(U), heg_s2=sc(U), dlog_nonce=sc(U),
               r_b_gamma=nm(alice), r_b_w=nm(alice), nb_gamma=sc(U), nbt_gamma=sc(U), nb_w=sc(U), nbt_w=sc(U), beta_tag_gamma=nm(alice), beta_tag_w=nm(alice))
    sig = gg18.sign_batch(engine, ks, 2, rows, w, ysig, msg, rnd)
    assert list(sig["status"]) == [0] * U
    assert all(_ecdsa_ok(sig["r"][e], sig["s"][e], ysig[e], msg[e]) for e in range(U))
    ks.free()
    # failure: the share party 4 sends to party 5 is off by one -> InvalidSS for receiver 5 only
    import mpecdsa_b200.keygen as kmod
    orig = kmod.vss_share

    def tampered(eng, t_, n_, polynomials):
        sh, cm = orig(eng, t_, n_, polynomials)
        sh[4][2] = (sh[4][2] + 1) % Q                                    # what party 4 sends to party 5 (index 3 of group 1)
        return sh, cm
    kmod.vss_share = tampered
    try:
        out3 = gg18.keygen_batch(engine, t, n, u, p_q, blind, polys, nonce)
    finally:
        kmod.vss_share = orig
    assert list(out3["status"]) == [0, 0, 0, 0, 0, pkg.ST_INVALID_SS]


@pytest.mark.gpu
def test_lindell17_bulk_parity_on_gpu(engine, pkg, keyset):
    """384 two-party signatures (random + boundary inputs: k = 1, k = q - 1, message = 0 and 2^256 - 1, rho = 0 and q^2 - 1, x2 = q - 1) against the
    oracle, bit for bit, every one verified by the reference's `verify` on the device and a sample under OpenSSL"""
    from mpecdsa_b200 import gg20, lindell17 as L
    rng = random.Random(0xB17C)
    n = 384
    c = _l17_case(keyset, rng, n)
    edge = [dict(k1=1), dict(k2=1), dict(k1=Q - 1, k2=Q - 1), dict(msg=0), dict(msg=(1 << 256) - 1), dict(rho=0), dict(rho=Q * Q - 1), dict(x2=Q - 1)]
    for i, e in enumerate(edge):
        for f, v in e.items():
            c[f][i] = v
    c["pub"] = [o.pt_mul(G, a * b % Q) for a, b in zip(c["x1"], c["x2"])]
    ks = gg20.KeySets(engine, [keyset])
    n_list = [keyset[r].dk.p * keyset[r].dk.q for r in range(3)]
    R1, R2 = engine.secp_mul(None, c["k1"]), engine.secp_mul(None, c["k2"])
    c3, st = L.p2_partial_sig(engine, n_list, c["rows"], c["c_key"], c["x2"], c["k2"], R1, c["msg"], c["rho"], c["r_enc"])
    assert not st.any()
    r, s, rec, st = L.p1_sign(engine, ks, c["rows"], c3, c["k1"], R2)
    assert not st.any()
    assert not L.verify(engine, r, s, c["pub"], c["msg"]).any()
    for i in list(range(len(edge))) + list(range(len(edge), n, 7)):
        want_c3 = l17.p2_partial_sig(c["eks"][i], c["c_key"][i], c["x2"][i], c["k2"][i], R1[i], c["msg"][i], c["rho"][i], c["r_enc"][i])
        assert c3[i] == want_c3, i
        assert (r[i], s[i], int(rec[i])) == l17.p1_sign(c["dks"][i], want_c3, c["k1"][i], R2[i]), i
    assert all(_ecdsa_ok(r[i], s[i], c["pub"][i], c["msg"][i]) for i in range(0, n, 16))
    ks.free()


# ------------------------------------------------------------------------------------------------ the same tests on the edge key sets
@pytest.fixture(scope="module")
def edge_keysets():
    return fixtures.load_edge_keysets()


# _l17_case puts party one on row i % 3, so every one of the 9 edge rows is party one in some run of these tests
@pytest.mark.parametrize("edge", [0, 1, 2], ids=lambda k: f"edge{k}")
@pytest.mark.parametrize("test", [test_lindell17_kernels_on_host_harness, test_zk_pdl_kernels_on_host_harness], ids=lambda f: f.__name__)
def test_host_harness_on_edge_keysets(hh, edge_keysets, test, edge):
    """the Lindell-2017 and zk-PDL host-harness tests on each key set of keys_edge.json (2047-bit N, p < q, p/q close to 2
    and to 4, N at both ends of the accepted range)"""
    test(hh, edge_keysets[edge])


@pytest.mark.gpu
@pytest.mark.parametrize("edge", [0, 1, 2], ids=lambda k: f"edge{k}")
@pytest.mark.parametrize("test", [test_lindell17_on_gpu_matches_oracle, test_zk_pdl_on_gpu_matches_oracle, test_gg18_whole_signing_on_gpu,
                                  test_lindell17_full_key_gen_on_gpu, test_gg18_key_generation_then_signing_on_gpu,
                                  test_lindell17_bulk_parity_on_gpu], ids=lambda f: f.__name__)
def test_protocols_on_gpu_on_edge_keysets(engine, pkg, edge_keysets, test, edge):
    """the GPU protocol tests above on each key set of keys_edge.json: decrypt_dev (p1_sign, the zk-PDL prover), GG18's index
    bookkeeping over rows whose ciphertext and plaintext widths differ, and Lindell's key generation over 2047-bit N"""
    test(engine, pkg, edge_keysets[edge])


# ------------------------------------------------------------------------------------------------ edge key rows at the range tops
def test_l17_case_puts_party_one_on_every_edge_row():
    rows = {(lk.dk.p, lk.dk.q) for _, lk, _ in _edge_rows()}
    used = {(d.p, d.q) for ks in fixtures.load_edge_keysets() for d in _l17_case(ks, random.Random(0), 3)["dks"]}
    assert used == rows and len(rows) == 9
    assert any(p / q > 3.9 for p, q in used) and any(q / p > 3.9 for p, q in used) and sum(p < q for p, q in used) >= 3


def _wide_rho(p, q, base, rng, tries=256):
    """rho above q^2 with base + rho q < N, drawn `tries` times, keeping the draw whose plaintext m = base + rho q has the largest
    (m mod p) - (m mod q): the difference decrypt_finish has to bring into [0, q)"""
    m = lambda r: base + r * Q
    return max((rng.randrange(Q * Q, (p * q - base) // Q) for _ in range(tries)), key=lambda r: m(r) % p - m(r) % q)


@pytest.mark.gpu
def test_lindell17_range_tops_on_edge_rows(engine, pkg):
    """Every edge row as party one's key, with each value at the top of its sampling range: rho = q^2 - 1, x1 = floor(q/3) - 1,
    r_key = r_enc = N - 1, x2 = k1 = k2 = q - 1 (so k2^-1 = q - 1 as well) and the message 2^256 - 1.

    Honest plaintexts stay below q^3, under both Paillier primes, so the CRT tail of p1_sign's decrypt has nothing to correct.  So
    each row also gets a c3 from a party two whose rho lies above q^2: `PartialSig::compute` does not bound it, the signature is
    the same because rho q vanishes mod q, and rho is picked so that (m mod p) - (m mod q) is large (more than 3 q on the rows with
    p/q close to 4, where the tail needs its fourth addition of q)."""
    from mpecdsa_b200 import gg20, lindell17 as L
    rows = _edge_rows()
    rng = random.Random(0x17ED)
    x1, x2, k, msg, rho = Q // 3 - 1, Q - 1, Q - 1, (1 << 256) - 1, Q * Q - 1
    R = o.pt_mul(G, k)                                                     # k1 = k2: both ephemeral public shares
    pub = o.pt_mul(G, x1 * x2 % Q)
    eks = [o.EncryptionKey(lk.dk.p * lk.dk.q, (lk.dk.p * lk.dk.q) ** 2) for _, lk, _ in rows]
    n_list = [ek.n for ek in eks]
    c_key = [o.paillier_encrypt(ek, x1, ek.n - 1) for ek in eks]
    m = len(rows)
    c3, st = L.p2_partial_sig(engine, n_list, list(range(m)), c_key, [x2] * m, [k] * m, [R] * m, [msg] * m, [rho] * m, [n - 1 for n in n_list])
    assert not st.any()
    assert c3 == [l17.p2_partial_sig(ek, ck, x2, k, R, msg, rho, ek.n - 1) for ek, ck in zip(eks, c_key)]
    kinv = pow(k, -1, Q)
    base = x1 * (kinv * (o.pt_mul(R, k)[0] % Q * x2 % Q) % Q) + kinv * msg % Q   # x1 v + (k2^-1 m mod q)
    plain = [base + rho * Q] * m
    for (_, lk, shape), ek, ck in zip(rows, eks, c_key):
        p, q = lk.dk.p, lk.dk.q
        r_w = _wide_rho(p, q, base, rng)
        plain.append(base + r_w * Q)
        assert plain[-1] < ek.n and (p < 3 * q or plain[-1] % p - plain[-1] % q > 3 * q), shape
        c3.append(l17.p2_partial_sig(ek, ck, x2, k, R, msg, r_w, ek.n - 1))
    key_row = list(range(m)) * 2
    dks = [rows[i][1].dk for i in key_row]
    assert [o.paillier_decrypt(d, c) for d, c in zip(dks, c3)] == plain
    edge = fixtures.load_edge_keysets()
    ks = gg20.KeySets(engine, edge)
    try:
        r, s, rec, st = L.p1_sign(engine, ks, key_row, c3, [k] * 2 * m, [R] * 2 * m)
    finally:
        ks.free()
    want = [l17.p1_sign(d, c, k, R) for d, c in zip(dks, c3)]
    wrong = [(rows[i][2], j >= m) for j, i in enumerate(key_row) if (r[j], s[j], int(rec[j])) != want[j]]
    assert not st.any() and wrong == []
    assert all(l17.verify(r[j], s[j], pub, msg) for j in range(2 * m)) and _ecdsa_ok(r[0], s[0], pub, msg)
    assert not L.verify(engine, r, s, [pub] * 2 * m, [msg] * 2 * m).any()


@pytest.mark.gpu
def test_zk_pdl_range_tops_on_edge_rows(engine, pkg):
    """Every edge row through the four messages with a = q - 1 and b = q^2 - 1, so that a + (b << bit_length(a)) has its largest
    width, x1 = floor(q/3) - 1 and r = N - 1.  alpha = a x1 + b < q^3 again leaves the prover's CRT tail nothing to correct, so the
    prover also decrypts the c' of a verifier that did not follow message1: the plaintexts with (m mod p, m mod q) = (p - 1, 0) and
    (0, q - 1), the most the tail ever corrects (four additions of q on the rows with p/q close to 4)."""
    from mpecdsa_b200 import gg20, lindell17 as L
    rows = _edge_rows()
    m = len(rows)
    x1, a, b, blind = Q // 3 - 1, Q - 1, Q * Q - 1, Q - 1
    assert (a + (b << a.bit_length())).bit_length() == 768
    eks = [o.EncryptionKey(lk.dk.p * lk.dk.q, (lk.dk.p * lk.dk.q) ** 2) for _, lk, _ in rows]
    n_list = [ek.n for ek in eks]
    c_key = [o.paillier_encrypt(ek, x1, ek.n - 1) for ek in eks]
    Qpt = o.pt_mul(G, x1)
    ct, ctt, qt, st = L.pdl_verifier_message1(engine, n_list, list(range(m)), c_key, [Qpt] * m, [a] * m, [b] * m, [n - 1 for n in n_list], [blind] * m)
    want = [l17.pdl_verifier_message1(ek, ck, Qpt, a, b, ek.n - 1, blind) for ek, ck in zip(eks, c_key)]
    assert not st.any() and ct == [w.c_tag for w in want] and ctt == [w.c_tag_tag for w in want] and qt == [w.q_tag for w in want]
    key_row, c_tag, plain = list(range(m)), list(ct), [a * x1 + b] * m
    for i, (_, lk, _) in enumerate(rows):
        for pl in _worst_plaintexts(lk.dk.p, lk.dk.q):
            key_row.append(i); c_tag.append(o.paillier_encrypt(eks[i], pl, eks[i].n - 1)); plain.append(pl)
    edge = fixtures.load_edge_keysets()
    ks = gg20.KeySets(engine, edge)
    try:
        ch, qh, al, st = L.pdl_prover_message1(engine, ks, key_row, c_tag, [blind] * len(c_tag))
    finally:
        ks.free()
    want_p = [l17.pdl_prover_message1(rows[i][1].dk, c, blind) for i, c in zip(key_row, c_tag)]
    assert [w[2] for w in want_p] == plain
    wrong = [(rows[i][2], j >= m) for j, i in enumerate(key_row) if (ch[j], qh[j], al[j]) != want_p[j]]
    assert not st.any() and wrong == []
    assert list(L.pdl_prover_message2(engine, [x1] * m, al[:m], ctt, [a] * m, [b] * m, [blind] * m)) == [0] * m
    assert list(L.pdl_verifier_finalize(engine, ch[:m], qh[:m], [blind] * m, qt)) == [0] * m


@pytest.mark.gpu
def test_lindell17_paillier_key_size_rule(engine, pkg):
    """Party two's `verify_ni_proof_correct_key` refuses `ek.n.bit_length() < PAILLIER_KEY_SIZE - 1` before it looks at the proof
    (party_two.rs:307): party one's 2047-bit moduli pass p2_verify_paillier_and_proofs, and a 2046-bit N whose NiCorrectKeyProof
    is valid gets IncorrectProof."""
    from mpecdsa_b200 import gg20, keygen, lindell17 as L
    edge = fixtures.load_edge_keysets()[0]
    raw = fixtures.edge_keysets_raw()[0]["parties"]
    rng = random.Random(0x2046)
    small = (prime_in(HALF, HALF + SLACK, rng), prime_in(HALF >> 1, (HALF >> 1) + SLACK, rng))
    # elements 0 and 1: rows 0 and 1 of edge key set 0; element 2 hands in the 2046-bit key (its PDL proof runs under row 2's key,
    # which does not matter: the size rule decides first)
    p_q = [(edge[i].dk.p, edge[i].dk.q) for i in range(2)] + [small]
    n_list = [p * q for p, q in p_q]
    assert [n.bit_length() for n in n_list] == [2047, 2047, 2046]
    stm = [(edge[i].h1_h2_n_tilde_vec[i].N, edge[i].h1_h2_n_tilde_vec[i].g, edge[i].h1_h2_n_tilde_vec[i].ni) for i in range(3)]
    # the CompositeDLogProof of (N~, h1, h2) is for the negated exponent phi(N~) - xhi (see keygen_oracle.h1_h2_n_tilde)
    H = lambda r, k: int(r[k], 16)
    neg_xhi = [(H(r, "p_tilde") - 1) * (H(r, "q_tilde") - 1) - H(r, "xhi") for r in raw]
    x1 = [Q // 3 - 1] + [rng.randrange(1, Q // 3) for _ in range(2)]
    pdl_rand = ([rng.randrange(Q ** 3) for _ in range(3)], [rng.randrange(1, n) for n in n_list], [rng.randrange(Q * s[0]) for s in stm],
                [rng.randrange(Q ** 3 * s[0]) for s in stm])
    ks = gg20.KeySets(engine, [edge])
    try:
        msg = L.p1_paillier_and_proofs(engine, ks, [0, 1, 2], [0, 1, 2], stm, neg_xhi, x1, [n - 1 for n in n_list], pdl_rand,
                                       [rng.getrandbits(500) for _ in range(3)], p_q)
        assert msg["correct_key_proof"] == [kg.correct_key_proof(o.DecryptionKey(p, q)) for p, q in p_q]
        assert all(kg.correct_key_verify(sv, o.EncryptionKey(n, n * n)) for sv, n in zip(msg["correct_key_proof"], n_list))
        assert list(keygen.correct_key_verify(engine, n_list, msg["correct_key_proof"])) == [0, 0, 0]
        assert all(kg.composite_dlog_verify(kg.CompositeDLogProof(*pf), o.DLogStatement(*s_)) for pf, s_ in zip(msg["composite_dlog_proof"], stm))
        st = L.p2_verify_paillier_and_proofs(engine, ks, [0, 1, 2], [0, 1, 2], stm, n_list, msg, msg["Q"])
    finally:
        ks.free()
    assert list(st) == [0, 0, pkg.ST_PROOF]
