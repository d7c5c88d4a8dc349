"""Keys at the edges of the domain the reference's keygen accepts (tests/golden/keys_edge.json): Paillier N and N~ of 2047
bits, p < q, p/q close to 2 and close to 4, N just above 2^2046 and just below 2^2048, h1 well below N~.

CPU: the fixtures are what they claim to be, and the Paillier CRT tails (decrypt_finish, crt_combine) compiled for the host
give the right value on every edge row for the inputs that need the most correction steps.
GPU: key upload, L1 Paillier, L2 proofs, keygen proofs and the offline stage over the edge key sets against the oracle or its
C twin, keys outside the domain refused, and verifier inputs that the reference accepts at the edge of their ABI slots."""
import ctypes
import dataclasses
import os
import random

import numpy as np
import pytest

from oracle import gg20_oracle as o
from oracle import keygen_oracle as kg
from oracle.sampling import Drbg, sample_unit
from tests.golden import fixtures
from tests.golden.make_edge_keys import MID, is_probable_prime
from tests.test_glue_host import KEY_SIZE, I, L, P, h  # noqa: F401  (h: the host harness fixture)

Q3 = o.Q ** 3
# (nearly) the largest alpha for which s1 = e*a + alpha <= q^3 for every challenge e < 2^256 and a < q: the reference's verifiers reject
# s1 > q^3 (range_proofs.rs:118), so a prover drawing alpha = q^3 - 1 with a = q - 1 is rejected by an honest verifier
# MtA's beta' < N: a*b + beta' must stay below N for Alice to decrypt a*b + beta' (mta/mod.rs:165), so the top is N - q^2
BETA_TAG_TOP = lambda n: n - o.Q ** 2
ALPHA_TOP = Q3 - (o.Q << 256) - 1           # - 1: alpha mod q != 0, so BobProofExt's u = alpha G is not the identity


def _rows():
    return [lk for ks in fixtures.load_edge_keysets() for lk in ks]


def _worst_plaintexts(p, q):
    """m with (m mod p, m mod q) = (p-1, 0) and (0, q-1): the most negative and the largest mq - mp of decrypt_finish"""
    n = p * q
    return [(p - 1) * q * pow(q, -1, p) % n, (q - 1) * p * pow(p, -1, q) % n]


def _crt(yp, yq, p, q):
    pp, qq = p * p, q * q
    return yp + pp * ((yq - yp) * pow(pp, -1, qq) % qq)


# ------------------------------------------------------------------------------------------------ CPU: fixtures
def test_edge_fixtures_are_prime_and_cover_the_domain():
    raw = fixtures.edge_keysets_raw()
    rng = random.Random(0xED6E)
    rows = [p for ks in raw for p in ks["parties"]]
    assert len(raw) == 3 and len(rows) == 9
    H = lambda s: int(s, 16)
    for r in rows:
        p, q, pt, qt, nt, h1, h2, xhi = (H(r[k]) for k in ("p", "q", "p_tilde", "q_tilde", "n_tilde", "h1", "h2", "xhi"))
        for x in (p, q, pt, qt):
            assert is_probable_prime(x, rng)
        n = p * q
        # the domain tecdsa_keys_upload accepts, and the bit-length checks of the reference's keygen
        assert p != q and p < 1 << 1024 and q < 1 << 1024 and 1 << 2046 <= n < 1 << 2048
        assert pt * qt == nt and 1 << 2046 <= nt < 1 << 2048
        assert kg.PAILLIER_MIN_BIT_LENGTH <= n.bit_length() <= kg.PAILLIER_MAX_BIT_LENGTH
        assert kg.PAILLIER_MIN_BIT_LENGTH <= nt.bit_length() <= kg.PAILLIER_MAX_BIT_LENGTH
        assert h2 == pow(h1, xhi, nt) and kg.h1_h2_n_tilde(pt, qt, h1, xhi)[:3] == (nt, h1, h2)
    for ks in raw:
        assert sorted({H(r["n_tilde"]).bit_length() for r in ks["parties"]}) == [2047, 2048]      # both N~ sizes in every key set
        x = [H(r["x_i"]) for r in ks["parties"]]                                                  # Feldman shares of a line
        assert (2 * x[0] - x[1]) % o.Q == H(ks["secret"]) and (x[2] - 2 * x[1] + x[0]) % o.Q == 0
    pq = [(H(r["p"]), H(r["q"])) for r in rows]
    N = [p * q for p, q in pq]
    assert any(n.bit_length() == 2047 and all(1 << 1023 <= f < MID for f in (p, q))
               and (p * p).bit_length() == (q * q).bit_length() == 2047 for (p, q), n in zip(pq, N))
    assert any(p < q for p, q in pq) and any(p > q for p, q in pq)
    assert any(1.9 < p / q < 2 and p.bit_length() == q.bit_length() == 1024 for p, q in pq)
    unbalanced = [(p, q) for p, q in pq if p.bit_length() == 1024 and q.bit_length() == 1023 and p / q > 3.9]
    assert unbalanced and all((p * q).bit_length() == 2047 for p, q in unbalanced)
    assert any(q / p > 3.9 for p, q in pq)
    assert min(N) < (1 << 2046) + (1 << 2030) and max(N) > (1 << 2048) - (1 << 2030)
    assert any(H(r["h1"]).bit_length() <= 1200 for r in rows)


def test_edge_fixtures_regenerate_identically():
    from tests.golden import make_edge_keys as mk
    raw = fixtures.edge_keysets_raw()
    assert mk.make_keyset(1, mk.KEYSETS[1]) == raw[1]


# ------------------------------------------------------------------------------------------------ CPU: CRT tails on the host
def test_host_crt_tails_on_edge_rows(h):
    """decrypt_finish and crt_combine (csrc/gg20_glue.cuh) on every edge row, at the inputs that need the most additions of q
    (resp. q^2): with p/q close to 4 the old bounds of 3 and 5 additions left the value negative."""
    rows = _rows()
    tabs = [np.zeros((len(rows), s), np.uint32) for s in KEY_SIZE]
    for r, lk in enumerate(rows):
        tabs[9][r] = L(lk.dk.p, 32); tabs[10][r] = L(lk.dk.q, 32)
    ptrs = (ctypes.c_void_p * len(tabs))(*[t.ctypes.data for t in tabs])
    h.h_key_setup(ptrs, len(rows))
    R, R64 = 1 << 1024, 1 << 2048
    rng = random.Random(0xC27)
    for r, lk in enumerate(rows):
        p, q = lk.dk.p, lk.dk.q
        n = p * q
        assert I(tabs[0][r]) == n and I(tabs[1][r]) == n * n and I(tabs[5][r]) == p * p and I(tabs[6][r]) == q * q
        assert I(tabs[11][r]) == pow(p, -1, R) and I(tabs[12][r]) == pow(q, -1, R)
        assert I(tabs[13][r]) == (-pow(q, -1, p)) % p * R % p and I(tabs[14][r]) == (-pow(p, -1, q)) % q * R % q
        assert I(tabs[15][r]) == pow(p, -1, q) * R % q and I(tabs[16][r]) == pow(p * p, -1, q * q) * R64 % (q * q)
        assert I(tabs[17][r]) == q % (p - 1) and I(tabs[18][r]) == p % (q - 1)
        pp, qq = p * p, q * q
        out = np.zeros(128, np.uint32)
        for yp, yq in [(pp - 1, 0), (0, qq - 1), (pp - 1, qq - 1), (0, 0), (pp - 1, 1)] + [(rng.randrange(pp), rng.randrange(qq)) for _ in range(6)]:
            h.h_crt_combine(P(out), ptrs, r, P(L(yp, 64)), P(L(yq, 64)))
            assert I(out) == _crt(yp, yq, p, q), (r, hex(yp)[:10], hex(yq)[:10])
        ek = o.EncryptionKey(n, n * n)
        out = np.zeros(64, np.uint32)
        for m in _worst_plaintexts(p, q) + [0, 1, n - 1] + [rng.randrange(n) for _ in range(4)]:
            c = o.paillier_encrypt(ek, m, rng.randrange(1, n))
            dp, dq = pow(c % pp, p - 1, pp), pow(c % qq, q - 1, qq)
            h.h_decrypt_finish(P(out), ptrs, r, P(L(dp, 64)), P(L(dq, 64)))
            assert I(out) == m, (r, m % p == p - 1, m % q == q - 1)


# ------------------------------------------------------------------------------------------------ GPU helpers
def _top_unit(keys, s_l, pos) -> o.UnitRandomness:
    """`sample_unit` with every value at the top of its reference range: scalars Q-1, r and beta N-1, gamma Q^3 N~-1,
    rho Q N~-1, PDL alpha Q^3-1 (PDL beta: sample_range(1, N-1) tops out at N-2); the range proofs' alpha is ALPHA_TOP"""
    lk = keys[pos]
    l_s = [x - 1 for x in s_l]
    n_own = lk.paillier_key_vec[lk.i - 1].n
    n_peer = lk.paillier_key_vec[l_s[1 - pos]].n
    top = o.Q - 1
    r = o.UnitRandomness()
    r.gamma_i = r.k_i = top
    r.blind = (1 << 256) - 1
    r.r_k = n_own - 1
    r.alice = [(ALPHA_TOP, n_own - 1, Q3 * st.N - 1, o.Q * st.N - 1) for st in lk.h1_h2_n_tilde_vec]
    r.r_gamma = r.r_w = n_peer - 1
    r.beta_tag_gamma = r.beta_tag_w = BETA_TAG_TOP(n_peer)
    r.nonce_gamma_b = r.nonce_gamma_beta = r.nonce_w_b = r.nonce_w_beta = top
    r.l = r.ped_s1 = r.ped_s2 = r.heg_s1 = r.heg_s2 = top
    st = lk.h1_h2_n_tilde_vec[l_s[1 - pos]]
    r.pdl = (Q3 - 1, n_own - 2, o.Q * st.N - 1, Q3 * st.N - 1)
    return r


@pytest.fixture(scope="module")
def edge():
    return fixtures.load_edge_keysets()


@pytest.fixture
def edge_ks(engine, edge):
    from mpecdsa_b200 import gg20
    ks = gg20.KeySets(engine, edge)
    yield ks
    ks.free()


def _ek(row):
    n = row.dk.p * row.dk.q
    return o.EncryptionKey(n, n * n)


def _st(row):
    return row.h1_h2_n_tilde_vec[row.i - 1]


# ------------------------------------------------------------------------------------------------ GPU: key upload
@pytest.mark.gpu
def test_edge_key_tables_derived_on_device(engine, edge_ks):
    rows = _rows()
    R, R64 = 1 << 1024, 1 << 2048
    assert edge_ks.table(0, 64) == [k.dk.p * k.dk.q for k in rows]
    assert edge_ks.table(1, 128) == [(k.dk.p * k.dk.q) ** 2 for k in rows]
    assert edge_ks.table(5, 64) == [k.dk.p ** 2 for k in rows]
    assert edge_ks.table(6, 64) == [k.dk.q ** 2 for k in rows]
    assert edge_ks.table(11, 32) == [pow(k.dk.p, -1, R) for k in rows]
    assert edge_ks.table(13, 32) == [(-pow(k.dk.q, -1, k.dk.p)) % k.dk.p * R % k.dk.p for k in rows]
    assert edge_ks.table(14, 32) == [(-pow(k.dk.p, -1, k.dk.q)) % k.dk.q * R % k.dk.q for k in rows]
    assert edge_ks.table(15, 32) == [pow(k.dk.p, -1, k.dk.q) * R % k.dk.q for k in rows]
    assert edge_ks.table(16, 64) == [pow(k.dk.p ** 2, -1, k.dk.q ** 2) * R64 % k.dk.q ** 2 for k in rows]


@pytest.mark.gpu
def test_upload_refuses_keys_outside_the_domain(engine, pkg, edge):
    """2046-bit N (gg_2020/test.rs:765 `test_small_paillier`), p == q, a 2046-bit N~ and an even modulus are refused with
    TECDSA_E_ARG before anything is allocated; the same key set with the row restored uploads."""
    import copy
    from mpecdsa_b200 import gg20
    raw = fixtures.edge_keysets_raw()
    shapes = {r["shape"]: (int(r["p"], 16), int(r["q"], 16)) for ks in raw for r in ks["parties"]}
    small = shapes["min_n"][0] * shapes["unbalanced"][1]                       # two primes near 2^1023 and 2^1022
    assert small.bit_length() == 2046
    base = edge[0]

    def with_row0(**kw):
        ks = copy.deepcopy(base)
        lk = ks[0]
        if "pq" in kw:
            lk.dk = o.DecryptionKey(*kw["pq"])
        if "nt" in kw:
            st = lk.h1_h2_n_tilde_vec[0]
            lk.h1_h2_n_tilde_vec[0] = o.DLogStatement(kw["nt"], st.g % kw["nt"], st.ni % kw["nt"])
        return ks

    p0 = base[0].dk.p
    bad = [with_row0(pq=(shapes["min_n"][0], shapes["unbalanced"][1])), with_row0(pq=(p0, p0)),
           with_row0(nt=int(raw[0]["parties"][0]["p_tilde"], 16) * shapes["unbalanced"][1]),
           with_row0(pq=(p0 + 1, base[0].dk.q))]
    assert bad[2][0].h1_h2_n_tilde_vec[0].N.bit_length() == 2046
    for ks in bad:
        with pytest.raises(pkg.EngineError, match=r"keys_upload.*rc=-1"):
            gg20.KeySets(engine, [edge[1], ks])
    ok = gg20.KeySets(engine, [edge[1], base])
    assert ok.table(0, 64)[3] == base[0].dk.p * base[0].dk.q
    ok.free()


# ------------------------------------------------------------------------------------------------ GPU: L1
@pytest.mark.gpu
def test_paillier_round_trip_on_edge_rows(engine, edge_ks):
    rows = _rows()
    rng = random.Random(0xED61)
    idx, m, r = [], [], []
    for i, lk in enumerate(rows):
        n = lk.dk.p * lk.dk.q
        for mm in _worst_plaintexts(lk.dk.p, lk.dk.q) + [0, 1, n - 1, rng.randrange(n)]:
            idx.append(i); m.append(mm); r.append(n - 1 if len(idx) % 2 else rng.randrange(1, n))
    ns = [lk.dk.p * lk.dk.q for lk in rows]
    eks = [_ek(lk) for lk in rows]
    c = engine.paillier_encrypt(ns, idx, m, r)
    assert c == [o.paillier_encrypt(eks[i], mm, rr) for i, mm, rr in zip(idx, m, r)]
    assert engine.paillier_decrypt(edge_ks.handle, idx, c) == m
    k = [o.Q - 1 if j % 3 == 0 else rng.randrange(o.Q) for j in range(len(idx))]
    ck = engine.paillier_mul(ns, idx, c, k)
    assert ck == [pow(cc, kk, eks[i].nn) for i, cc, kk in zip(idx, c, k)]
    cs = engine.paillier_add(ns, idx, c, ck)
    assert cs == [x * y % eks[i].nn for i, x, y in zip(idx, c, ck)]
    dec = engine.paillier_decrypt(edge_ks.handle, idx, cs)
    assert dec == [(mm + mm * kk) % ns[i] for i, mm, kk in zip(idx, m, k)]
    assert dec == [o.paillier_decrypt(rows[i].dk, x) for i, x in zip(idx, cs)]


# ------------------------------------------------------------------------------------------------ GPU: L2
def _l2_instances(n_rows):
    """(ek_row, st_row, top) triples: every edge row as prover key and as statement, once at the top of the ranges and once
    with random values"""
    return [(i, (i + 1) % n_rows, True) for i in range(n_rows)] + [(i, (i + 5) % n_rows, False) for i in range(n_rows)]


def _range_status(pkg, accepted):
    return [0 if ok else pkg.ST_RANGE for ok in accepted]


@pytest.mark.gpu
def test_alice_bob_pdl_proofs_on_edge_rows(engine, pkg, edge_ks):
    from mpecdsa_b200 import gg20
    rows = _rows()
    inst = _l2_instances(len(rows))
    er, sr = [i[0] for i in inst], [i[1] for i in inst]
    rng = Drbg(0xED62, "edge-l2")
    # AliceProof
    a, r, c, al, be, ga, ro = [], [], [], [], [], [], []
    for e_i, s_i, top in inst:
        ek, st = _ek(rows[e_i]), _st(rows[s_i])
        if top:
            vals = (o.Q - 1, ek.n - 1, ALPHA_TOP, ek.n - 1, Q3 * st.N - 1, o.Q * st.N - 1)
        else:
            vals = (rng.scalar(), rng.unit_mod(ek.n), rng.below(Q3), rng.unit_mod(ek.n), rng.below(Q3 * st.N), rng.below(o.Q * st.N))
        for lst, v in zip((a, r, al, be, ga, ro), vals):
            lst.append(v)
        c.append(o.paillier_encrypt(ek, a[-1], r[-1]))
    pf = gg20.alice_proof_generate(engine, edge_ks, er, sr, a, c, r, al, be, ga, ro)
    for j, (e_i, s_i, _) in enumerate(inst):
        w = o.alice_proof_generate(a[j], c[j], _ek(rows[e_i]), _st(rows[s_i]), r[j], al[j], be[j], ga[j], ro[j])
        assert (pf["z"][j], pf["e"][j], pf["s"][j], pf["s1"][j], pf["s2"][j]) == (w.z, w.e, w.s, w.s1, w.s2), j
        assert o.alice_proof_verify(w, c[j], _ek(rows[e_i]), _st(rows[s_i]))
    assert not gg20.alice_proof_verify(engine, edge_ks, er, sr, c, pf["z"], pf["e"], pf["s"], pf["s1"], pf["s2"]).any()
    # alpha = q^3 - 1 with a = q - 1: s1 > q^3, rejected by the oracle and by the GPU with the range status
    top = [j for j, i in enumerate(inst) if i[2]]
    al2 = [Q3 - 1 if j in top else v for j, v in enumerate(al)]
    pf2 = gg20.alice_proof_generate(engine, edge_ks, er, sr, a, c, r, al2, be, ga, ro)
    acc = [o.alice_proof_verify(o.alice_proof_generate(a[j], c[j], _ek(rows[e_i]), _st(rows[s_i]), r[j], al2[j], be[j], ga[j], ro[j]),
                                c[j], _ek(rows[e_i]), _st(rows[s_i])) for j, (e_i, s_i, _) in enumerate(inst)]
    assert not any(acc[j] for j in top) and all(acc[j] for j in range(len(inst)) if j not in top)
    assert list(gg20.alice_proof_verify(engine, edge_ks, er, sr, c, pf2["z"], pf2["e"], pf2["s"], pf2["s1"], pf2["s2"])) == _range_status(pkg, acc)
    # BobProof and BobProofExt
    for check in (False, True):
        cols = {k: [] for k in ("a_enc", "mta", "b", "bp", "r", "al", "be", "ga", "ro", "rp", "si", "ta")}
        for e_i, s_i, top in inst:
            ek, st = _ek(rows[e_i]), _st(rows[s_i])
            enc_a = o.paillier_encrypt(ek, rng.scalar(), rng.unit_mod(ek.n))
            if top:
                b, bp, rr = o.Q - 1, ek.n - 1, ek.n - 1
                rest = (ALPHA_TOP, ek.n - 1, o.Q ** 2 * ek.n - 1, o.Q * st.N - 1, Q3 * st.N - 1, o.Q * st.N - 1, Q3 * st.N - 1)
            else:
                b, bp, rr = rng.scalar(), rng.below(ek.n), rng.unit_mod(ek.n)
                rest = (rng.below(Q3), rng.unit_mod(ek.n), rng.below(o.Q ** 2 * ek.n), rng.below(o.Q * st.N), rng.below(Q3 * st.N),
                        rng.below(o.Q * st.N), rng.below(Q3 * st.N))
            mta = o.paillier_add(ek, o.paillier_mul(ek, enc_a, b), o.paillier_encrypt(ek, bp, rr))
            for k, v in zip(cols, (enc_a, mta, b, bp, rr) + rest):
                cols[k].append(v)
        bpf = gg20.bob_proof_generate(engine, edge_ks, er, sr, check, *[cols[k] for k in cols])
        Xs = [o.pt_mul(o.G, b) for b in cols["b"]]
        for j, (e_i, s_i, _) in enumerate(inst):
            ek, st = _ek(rows[e_i]), _st(rows[s_i])
            w, u = o.bob_proof_generate(cols["a_enc"][j], cols["mta"][j], cols["b"][j], cols["bp"][j], ek, st, cols["r"][j], check,
                                        *[cols[k][j] for k in ("al", "be", "ga", "ro", "rp", "si", "ta")])
            assert tuple(bpf[k][j] for k in ("t", "z", "e", "s", "s1", "s2", "t1", "t2")) == (w.t, w.z, w.e, w.s, w.s1, w.s2, w.t1, w.t2), (check, j)
            assert (o.bob_proof_ext_verify(w, u, cols["a_enc"][j], cols["mta"][j], ek, st, Xs[j]) if check
                    else o.bob_proof_verify(w, cols["a_enc"][j], cols["mta"][j], ek, st))
        st_ok = gg20.bob_proof_verify(engine, edge_ks, er, sr, cols["a_enc"], cols["mta"], bpf, Xs if check else None, bpf["u"] if check else None)
        assert not st_ok.any(), check
    # PDLwSlack
    x, r, c, Qs, Gs, al, be, rh, ga = ([] for _ in range(9))
    for e_i, s_i, top in inst:
        ek, st = _ek(rows[e_i]), _st(rows[s_i])
        if top:
            vals = (o.Q - 1, ek.n - 1, Q3 - 1, ek.n - 2, o.Q * st.N - 1, Q3 * st.N - 1)
        else:
            vals = (rng.scalar(), rng.unit_mod(ek.n), rng.below(Q3), 1 + rng.below(ek.n - 2), rng.below(o.Q * st.N), rng.below(Q3 * st.N))
        for lst, v in zip((x, r, al, be, rh, ga), vals):
            lst.append(v)
        c.append(o.paillier_encrypt(ek, x[-1], r[-1]))
        Gs.append(o.pt_mul(o.G, rng.scalar())); Qs.append(o.pt_mul(Gs[-1], x[-1]))
    ppf = gg20.pdl_prove(engine, edge_ks, er, sr, x, r, c, Qs, Gs, al, be, rh, ga)
    for j, (e_i, s_i, _) in enumerate(inst):
        ek, st = _ek(rows[e_i]), _st(rows[s_i])
        w = o.pdl_prove(x[j], r[j], c[j], ek, Qs[j], Gs[j], st.g, st.ni, st.N, al[j], be[j], rh[j], ga[j])
        assert tuple(ppf[k][j] for k in ("z", "u1", "u2", "u3", "s1", "s2", "s3")) == (w.z, w.u1, w.u2, w.u3, w.s1, w.s2, w.s3), j
    assert not gg20.pdl_verify(engine, edge_ks, er, sr, c, Qs, Gs, *[ppf[k] for k in ("z", "u1", "u2", "u3", "s1", "s2", "s3")]).any()


@pytest.mark.gpu
def test_mta_on_edge_rows(engine, pkg, edge_ks):
    from mpecdsa_b200 import gg20
    rows = _rows()
    n = len(rows) * 2
    ek_row = [i % len(rows) for i in range(n)]
    st_rows = [[3 * (e // 3) + x for x in range(3)] for e in ek_row]     # the key set's whole h1_h2_n_tilde_vec
    top = [i < len(rows) for i in range(n)]
    rng = Drbg(0xED63, "edge-mta")
    a, r, pr = [], [], []
    for i in range(n):
        ek = _ek(rows[ek_row[i]])
        stmts = [_st(rows[s]) for s in st_rows[i]]
        if top[i]:
            a.append(o.Q - 1); r.append(ek.n - 1)
            pr.append([(ALPHA_TOP, ek.n - 1, Q3 * st.N - 1, o.Q * st.N - 1) for st in stmts])
        else:
            a.append(rng.scalar()); r.append(rng.below(ek.n))
            pr.append([(rng.below(Q3), rng.unit_mod(ek.n), rng.below(Q3 * st.N), rng.below(o.Q * st.N)) for st in stmts])
    c, proofs = gg20.mta_message_a(engine, edge_ks, ek_row, st_rows, a, r, pr)
    m_as = []
    for i in range(n):
        m_a = o.message_a(a[i], _ek(rows[ek_row[i]]), r[i], [_st(rows[s]) for s in st_rows[i]], pr[i])
        m_as.append(m_a)
        assert c[i] == m_a.c
        for x, pf in enumerate(m_a.range_proofs):
            assert tuple(proofs[k][i][x] for k in ("z", "e", "s", "s1", "s2")) == (pf.z, pf.e, pf.s, pf.s1, pf.s2)
    # every range proof of MessageA verifies through the L2 entry point as well
    flat_er = [e for e in ek_row for _ in range(3)]
    flat_sr = [s for row in st_rows for s in row]
    got = gg20.alice_proof_verify(engine, edge_ks, flat_er, flat_sr, [x for x in c for _ in range(3)],
                                  *[[v for inst in proofs[k] for v in inst] for k in ("z", "e", "s", "s1", "s2")])
    assert list(got) == [0] * len(flat_er)
    b = [o.Q - 1 if top[i] else rng.scalar() for i in range(n)]
    rand_b = [_ek(rows[e]).n - 1 if top[i] else rng.below(_ek(rows[e]).n) for i, e in enumerate(ek_row)]
    beta_tag = [BETA_TAG_TOP(_ek(rows[e]).n) if top[i] else rng.below(_ek(rows[e]).n) for i, e in enumerate(ek_row)]
    nb = [o.Q - 1 if top[i] else rng.scalar() for i in range(n)]
    nbt = [o.Q - 1 if top[i] else rng.scalar() for i in range(n)]
    c_b, bp, btp, beta, st = gg20.mta_message_b(engine, edge_ks, ek_row, st_rows, b, c, proofs, rand_b, beta_tag, nb, nbt)
    want = [o.message_b(b[i], _ek(rows[ek_row[i]]), m_as[i], rand_b[i], beta_tag[i], [_st(rows[s]) for s in st_rows[i]], nb[i], nbt[i])
            for i in range(n)]
    assert [w is None for w in want] == [False] * n
    assert list(st) == [0] * n
    for i in range(n):
        m_b, beta_w = o.message_b(b[i], _ek(rows[ek_row[i]]), m_as[i], rand_b[i], beta_tag[i], [_st(rows[s]) for s in st_rows[i]], nb[i], nbt[i])
        assert c_b[i] == m_b.c and beta[i] == beta_w
    alpha, plain, st2 = gg20.mta_get_alpha(engine, edge_ks, ek_row, a, c_b, bp, btp)
    assert not st2.any()
    for i in range(n):
        assert (alpha[i] + beta[i]) % o.Q == a[i] * b[i] % o.Q
        assert plain[i] == o.paillier_decrypt(rows[ek_row[i]].dk, c_b[i])


# ------------------------------------------------------------------------------------------------ GPU: keygen
@pytest.mark.gpu
def test_keygen_proofs_on_edge_rows(engine, pkg):
    from mpecdsa_b200 import keygen
    raw = [r for ks in fixtures.edge_keysets_raw() for r in ks["parties"]]
    H = lambda s: int(s, 16)
    pq = [(H(r["p"]), H(r["q"])) for r in raw]
    assert {(p * q).bit_length() for p, q in pq} == {2047, 2048}
    sig, st = keygen.correct_key_prove(engine, pq)
    assert list(st) == [0] * len(pq)
    assert sig == [kg.correct_key_proof(o.DecryptionKey(p, q)) for p, q in pq]
    assert list(keygen.correct_key_verify(engine, [p * q for p, q in pq], sig)) == [0] * len(pq)
    bad = [list(s) for s in sig]
    bad[0][7] ^= 1                                     # the last mask digest of a 2047-bit row
    assert list(keygen.correct_key_verify(engine, [p * q for p, q in pq[:1]], bad[:1])) == [pkg.ST_PROOF]
    setups = [(H(r["p_tilde"]), H(r["q_tilde"]), H(r["h1"]), H(r["xhi"])) for r in raw]
    got, st = keygen.h1_h2_n_tilde(engine, setups)
    assert list(st) == [0] * len(setups)
    assert got == [kg.h1_h2_n_tilde(*s) for s in setups]
    assert [g[0] for g in got] == [H(r["n_tilde"]) for r in raw] and [g[2] for g in got] == [H(r["h2"]) for r in raw]
    rng = random.Random(0xED64)
    stmts, secrets, nonces, want = [], [], [], []
    for nt, h1, h2, xn, xin in got:
        for stmt, sec in (((nt, h1, h2), xn), ((nt, h2, h1), xin)):
            rr = rng.getrandbits(512) if len(nonces) % 2 else (1 << 512) - 1
            stmts.append(stmt); secrets.append(sec); nonces.append(rr)
            pf = kg.composite_dlog_prove(o.DLogStatement(*stmt), sec, rr)
            assert kg.composite_dlog_verify(pf, o.DLogStatement(*stmt))
            want.append((pf.x, pf.y))
    assert keygen.composite_dlog_prove(engine, stmts, secrets, nonces) == want
    assert list(keygen.composite_dlog_verify(engine, stmts, want)) == [0] * len(stmts)
    # the broadcast check: 2047-bit N and N~ pass, a 2046-bit N or N~ is a bad actor
    shapes = {r["shape"]: r for r in raw}
    small = H(shapes["min_n"]["p"]) * H(shapes["unbalanced"]["q"])
    p_small, q_small = H(shapes["min_n"]["p"]), H(shapes["unbalanced"]["q"])
    assert small.bit_length() == 2046
    cases = [(pq[0], setups[0]), (pq[5], setups[6]), ((p_small, q_small), setups[0]),
             (pq[1], (H(shapes["min_n"]["p_tilde"]), H(shapes["unbalanced"]["q"]), setups[1][2], setups[1][3]))]
    bcs, decs = [], []
    for (p, q), (pt, qt, h1, xhi) in cases:
        while True:
            try:
                pow(xhi, -1, (pt - 1) * (qt - 1))
                break
            except ValueError:
                xhi += 1
        nt, h1_, h2, xn, xin = kg.h1_h2_n_tilde(pt, qt, h1 % (pt * qt), xhi)
        y_i = o.pt_mul(o.G, rng.randrange(1, o.Q))
        bc, dec = kg.phase1_broadcast(o.DecryptionKey(p, q), nt, h1_, h2, xn, xin, y_i, rng.getrandbits(256), rng.getrandbits(512), rng.getrandbits(512))
        bcs.append(bc); decs.append(dec)
    assert [b.e.n.bit_length() for b in bcs][:3] == [(pq[0][0] * pq[0][1]).bit_length(), (pq[5][0] * pq[5][1]).bit_length(), 2046]
    assert bcs[3].dlog_statement.N.bit_length() == 2046
    want = [kg.phase1_verify(b, d) for b, d in zip(bcs, decs)]
    assert want == [True, True, False, False]
    assert list(keygen.phase1_verify(engine, bcs, decs)) == want


# ------------------------------------------------------------------------------------------------ GPU: offline stage
PAIRS = [(0, 1), (0, 2), (1, 2), (1, 0), (2, 0), (2, 1)]


@pytest.mark.gpu
@pytest.mark.parametrize("sampler", ["sample_unit", "top_of_range"])
def test_offline_every_signer_pair_matches_oracle(engine, pkg, edge, edge_ks, sampler):
    from mpecdsa_b200 import gg20
    rng = Drbg(0xED65, "edge-offline")
    sess, rnds, oracle_in = [], [], []
    for k, ks in enumerate(edge):
        for a, b in PAIRS:
            keys, s_l = [ks[a], ks[b]], [a + 1, b + 1]
            r = [sample_unit(rng, keys, s_l, p) if sampler == "sample_unit" else _top_unit(keys, s_l, p) for p in range(2)]
            sess.append((k, a, b)); rnds += r; oracle_in.append((keys, s_l, r))
    res = gg20.offline_batch(engine, edge_ks, sess, gg20.pack_randomness(rnds))
    for s, (keys, s_l, r) in enumerate(oracle_in):
        want = o.offline_session(keys, s_l, r)
        for p in range(2):
            u = 2 * s + p
            assert want[p].status == 0 and res.status[u] == 0, (sess[s], p)
            assert gg20.unpack_point(pkg.limbs_to_ints(res.R[u:u + 1])[0]) == want[p].R
            assert pkg.limbs_to_ints(res.sigma[u:u + 1])[0] == want[p].sigma_i, (sess[s], p)
            assert [gg20.unpack_point(v) for v in pkg.limbs_to_ints(res.t_vec[u].reshape(2, 16))] == want[p].t_vec
            assert int.from_bytes(res.digest[u].tobytes(), "little").to_bytes(32, "big") == want[p].transcript, (sess[s], p)


@pytest.mark.gpu
def test_split_batch_over_edge_and_standard_keysets_matches_twin(engine, edge):
    """2101 sessions over the 3 edge and the 8 standard key sets: the split driver, 2047- and 2048-bit rows mixed inside
    warps and sliding-window classes; every unit equals the C twin's."""
    from mpecdsa_b200 import gg20
    from oracle import twin
    keysets = edge + fixtures.load_all_keysets()
    sess, rnd = gg20.synthetic_batch(keysets, 2101, 0xED66)
    assert set(sess[:, 0].tolist()) == set(range(len(keysets)))
    ks = gg20.KeySets(engine, keysets)
    try:
        res = gg20.offline_batch(engine, ks, sess, rnd)
    finally:
        ks.free()
    tw = twin.offline_batch(twin.KeyTables(keysets), sess, rnd, os.cpu_count() or 1)
    assert not tw.status.any()
    assert np.array_equal(res.status, tw.status)
    for f in ("R", "sigma", "t_vec", "digest"):
        assert np.array_equal(getattr(res, f), getattr(tw, f)), f


@pytest.mark.gpu
def test_edge_signatures_verify_under_openssl(engine, pkg, edge, edge_ks):
    from cryptography.hazmat.primitives import hashes
    from cryptography.hazmat.primitives.asymmetric import ec, utils
    from mpecdsa_b200 import gg20
    rng = Drbg(0xED67, "edge-sign")
    sess = [(0, 0, 1), (1, 1, 2)]                     # the unbalanced row of key set 0 and the swapped one of key set 1
    rnds = []
    for k, a, b in sess:
        keys, s_l = [edge[k][a], edge[k][b]], [a + 1, b + 1]
        rnds += [sample_unit(rng, keys, s_l, p) for p in range(2)]
    res = gg20.offline_batch(engine, edge_ks, sess, gg20.pack_randomness(rnds))
    assert not res.status.any()
    msg = o.sha256_bigints([o.bn_from_bytes(b"edge keys")])
    for s, (k, _, _) in enumerate(sess):
        R = gg20.unpack_point(pkg.limbs_to_ints(res.R[2 * s:2 * s + 1])[0])
        parts = [o.local_sig(rnds[2 * s + p].k_i, msg, R, pkg.limbs_to_ints(res.sigma[2 * s + p:2 * s + p + 1])[0]) for p in range(2)]
        r_, s_, _ = o.output_signature(R, parts)
        y = edge[k][0].y_sum_s
        pub = ec.EllipticCurvePublicNumbers(y[0], y[1], ec.SECP256K1()).public_key()
        pub.verify(utils.encode_dss_signature(r_, s_), msg.to_bytes(32, "big"), ec.ECDSA(utils.Prehashed(hashes.SHA256())))


# ------------------------------------------------------------------------------------------------ GPU: verifier inputs at slot edges
@pytest.mark.gpu
def test_verifiers_accept_reference_valid_inputs_at_slot_edges(engine, pkg, edge_ks):
    """Proofs the reference accepts whose fields sit at the top of their ABI slots: s2 / t2 / s3 in [2^2943, 2^2944) (the
    windows 353-367 of the per-key fixed-base tables, which honest proofs never reach), s + N, a ciphertext c + N^2 hashed as
    such, and s1 = Q^3 exactly.  Each is accepted, and a one-bit change of the field is rejected with the oracle's status."""
    from mpecdsa_b200 import gg20
    rows = _rows()
    # s + N < 2^2048 and c + N^2 < 2^4096 need a 2047-bit N
    small = [i for i, lk in enumerate(rows) if (lk.dk.p * lk.dk.q).bit_length() == 2047]
    assert len(small) >= 3
    rng = Drbg(0xED68, "edge-slots")
    big = lambda: (1 << 2943) + rng.bits(2900)
    # AliceProof: kinds 0 big s2, 1 s + N, 2 c + N^2, 3 s1 = Q^3
    er, sr, cs, pfs = [], [], [], []
    for kind in range(4):
        for e_i in (small if kind in (1, 2) else range(len(rows))):
            s_i = (e_i + 4) % len(rows)
            ek, st = _ek(rows[e_i]), _st(rows[s_i])
            a, r = (0, rng.unit_mod(ek.n)) if kind == 3 else (rng.scalar(), rng.unit_mod(ek.n))
            c = o.paillier_encrypt(ek, a, r) + (ek.nn if kind == 2 else 0)
            gamma = big() if kind == 0 else rng.below(Q3 * st.N)
            pf = o.alice_proof_generate(a, c, ek, st, r, Q3 if kind == 3 else rng.below(Q3), rng.unit_mod(ek.n), gamma, rng.below(o.Q * st.N))
            if kind == 1:
                pf.s += ek.n
            assert pf.s < 1 << 2048 and c < 1 << 4096
            assert o.alice_proof_verify(pf, c, ek, st)
            assert (kind != 0 or pf.s2 >> 2943 == 1) and (kind != 3 or pf.s1 == Q3)
            er.append(e_i); sr.append(s_i); cs.append((kind, c)); pfs.append(pf)
    ver = lambda c, pfs: gg20.alice_proof_verify(engine, edge_ks, er, sr, c, [p.z for p in pfs], [p.e for p in pfs], [p.s for p in pfs],
                                                 [p.s1 for p in pfs], [p.s2 for p in pfs])
    assert not ver([c for _, c in cs], pfs).any()
    flipped, cflip, want = [], [], []
    for (kind, c), pf, e_i, s_i in zip(cs, pfs, er, sr):
        f = dataclasses.replace(pf)
        if kind == 0:
            f.s2 ^= 1 << 2943
        elif kind == 1:
            f.s ^= 1
        elif kind == 3:
            f.s1 += 1
        c2 = c ^ 1 if kind == 2 else c
        ok = o.alice_proof_verify(f, c2, _ek(rows[e_i]), _st(rows[s_i]))
        assert not ok
        flipped.append(f); cflip.append(c2)
        want.append(pkg.ST_RANGE if kind == 3 else pkg.ST_HASH_MISMATCH)
    assert list(ver(cflip, flipped)) == want
    # BobProofExt with t2 in [2^2943, 2^2944) (tau that large), and PDL with s3 there (gamma that large)
    n = len(rows)
    er, sr = list(range(n)), [(i + 2) % n for i in range(n)]
    cols = {k: [] for k in ("a_enc", "mta", "b")}
    bpfs, us = [], []
    for e_i, s_i in zip(er, sr):
        ek, st = _ek(rows[e_i]), _st(rows[s_i])
        enc_a = o.paillier_encrypt(ek, rng.scalar(), rng.unit_mod(ek.n))
        b, bp, r = rng.scalar(), rng.below(ek.n), rng.unit_mod(ek.n)
        mta = o.paillier_add(ek, o.paillier_mul(ek, enc_a, b), o.paillier_encrypt(ek, bp, r))
        w, u = o.bob_proof_generate(enc_a, mta, b, bp, ek, st, r, True, rng.below(Q3), rng.unit_mod(ek.n), rng.below(o.Q ** 2 * ek.n),
                                    rng.below(o.Q * st.N), rng.below(Q3 * st.N), rng.below(o.Q * st.N), big())
        assert w.t2 >> 2943 == 1 and o.bob_proof_ext_verify(w, u, enc_a, mta, ek, st, o.pt_mul(o.G, b))
        cols["a_enc"].append(enc_a); cols["mta"].append(mta); cols["b"].append(b); bpfs.append(w); us.append(u)
    Xs = [o.pt_mul(o.G, b) for b in cols["b"]]
    pfd = {k: [getattr(w, k) for w in bpfs] for k in ("t", "z", "e", "s", "s1", "s2", "t1", "t2")}
    assert not gg20.bob_proof_verify(engine, edge_ks, er, sr, cols["a_enc"], cols["mta"], pfd, Xs, us).any()
    pfd["t2"] = [v ^ (1 << 2943) for v in pfd["t2"]]
    assert list(gg20.bob_proof_verify(engine, edge_ks, er, sr, cols["a_enc"], cols["mta"], pfd, Xs, us)) == [pkg.ST_HASH_MISMATCH] * n
    pdl = []
    for e_i, s_i in zip(er, sr):
        ek, st = _ek(rows[e_i]), _st(rows[s_i])
        x, r = rng.scalar(), rng.unit_mod(ek.n)
        c = o.paillier_encrypt(ek, x, r)
        Gp = o.pt_mul(o.G, rng.scalar())
        Qp = o.pt_mul(Gp, x)
        w = o.pdl_prove(x, r, c, ek, Qp, Gp, st.g, st.ni, st.N, rng.below(Q3), 1 + rng.below(ek.n - 2), rng.below(o.Q * st.N), big())
        assert w.s3 >> 2943 == 1 and o.pdl_verify(w, c, ek, Qp, Gp, st.g, st.ni, st.N)
        pdl.append((c, Qp, Gp, w))
    args = lambda s3: ([c for c, _, _, _ in pdl], [q for _, q, _, _ in pdl], [g for _, _, g, _ in pdl], [w.z for *_, w in pdl],
                       [w.u1 for *_, w in pdl], [w.u2 for *_, w in pdl], [w.u3 for *_, w in pdl], [w.s1 for *_, w in pdl],
                       [w.s2 for *_, w in pdl], s3)
    assert not gg20.pdl_verify(engine, edge_ks, er, sr, *args([w.s3 for *_, w in pdl])).any()
    s3_bad = [w.s3 ^ (1 << 2943) for *_, w in pdl]
    for (c, Qp, Gp, w), s3, e_i, s_i in zip(pdl, s3_bad, er, sr):
        st = _st(rows[s_i])
        assert not o.pdl_verify(dataclasses.replace(w, s3=s3), c, _ek(rows[e_i]), Qp, Gp, st.g, st.ni, st.N)
    assert list(gg20.pdl_verify(engine, edge_ks, er, sr, *args(s3_bad))) == [pkg.ST_PDL_VERIFY] * n
