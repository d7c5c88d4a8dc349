"""Identifiable abort (SURVEY.md section 8(f) rank 3, /root/reference/src/protocols/multi_party_ecdsa/gg_2020/blame.rs): the oracle's
restatement on honest and corrupted three-signer transcripts (CPU), and the engine's batched re-derivation against it (GPU) —
the fault-injection style of gg_2020/test.rs:69-148 (`corrupt_step`), applied to the opened values."""
import copy
import random

import numpy as np
import pytest

from oracle import blame_oracle as bo
from oracle import gg20_oracle as o
from tests.golden import fixtures
from tests.test_edge_keys import _worst_plaintexts

Q = o.Q


def _transcript(keyset, seed=0xB1A):
    """An honest MtA / MtAwc transcript of three signers (every ordered pair plays Alice/Bob once) + everything phase 5-7 open"""
    rng = random.Random(seed)
    n = 3
    eks = [k.paillier_key_vec[k.i - 1] for k in keyset]
    dks = [k.dk for k in keyset]
    k = [rng.randrange(1, Q) for _ in range(n)]
    gamma = [rng.randrange(1, Q) for _ in range(n)]
    w = [rng.randrange(1, Q) for _ in range(n)]
    r_k = [rng.randrange(1, eks[i].n) for i in range(n)]
    c_a = [o.paillier_encrypt(eks[i], k[i], r_k[i]) for i in range(n)]
    beta_tag = [[rng.randrange(eks[i].n >> 1) for _ in range(n - 1)] for i in range(n)]          # [alice][j]: drawn by bob `ind`
    beta_rnd = [[rng.randrange(1, eks[i].n) for _ in range(n - 1)] for i in range(n)]
    nu_tag = [[rng.randrange(eks[i].n >> 1) for _ in range(n - 1)] for i in range(n)]
    nu_rnd = [[rng.randrange(1, eks[i].n) for _ in range(n - 1)] for i in range(n)]
    ind = lambda i, j: j if j < i else j + 1
    c_b = [[o.paillier_add(eks[i], o.paillier_mul(eks[i], c_a[i], gamma[ind(i, j)]), o.paillier_encrypt(eks[i], beta_tag[i][j], beta_rnd[i][j]))
            for j in range(n - 1)] for i in range(n)]
    c_bw = [[o.paillier_add(eks[i], o.paillier_mul(eks[i], c_a[i], w[ind(i, j)]), o.paillier_encrypt(eks[i], nu_tag[i][j], nu_rnd[i][j]))
             for j in range(n - 1)] for i in range(n)]
    alpha = [[(k[i] * gamma[ind(i, j)] + beta_tag[i][j]) % Q for j in range(n - 1)] for i in range(n)]
    beta = [[(-beta_tag[i][j]) % Q for j in range(n - 1)] for i in range(n)]
    delta, sigma = [], []
    miu = [[o.paillier_open(dks[i], c_bw[i][j]) for j in range(n - 1)] for i in range(n)]     # (plaintext before reduction, randomness)
    for i in range(n):
        d = k[i] * gamma[i] + sum(alpha[i])
        s = k[i] * w[i] + sum(m for m, _ in miu[i])
        for j in range(n - 1):
            i1, i2 = (j, i - 1) if j < i else (j + 1, i)
            d += beta[i1][i2]
            s += (-nu_tag[i1][i2]) % Q
        delta.append(d % Q); sigma.append(s % Q)
    R = o.pt_mul(o.G, pow(sum(k) % Q, -1, Q))            # any point works for the checks; this is R of an honest run with delta = k gamma
    S = [o.pt_mul(R, s) for s in sigma]
    nonces = [rng.randrange(1, Q) for _ in range(n)]
    proofs = [o.ecddh_prove(sigma[i], o.G, o.pt_mul(o.G, sigma[i]), R, S[i], nonces[i]) for i in range(n)]
    m = rng.getrandbits(256)
    r = R[0] % Q
    s_vec = [(m % Q * k[i] + r * sigma[i]) % Q for i in range(n)]
    p5 = bo.GlobalStatePhase5(k, r_k, gamma, beta_rnd, beta_tag, eks, delta, [o.pt_mul(o.G, g) for g in gamma], c_a, c_b)
    p6 = bo.GlobalStatePhase6(k, r_k, [[x[0] for x in row] for row in miu], [[x[1] for x in row] for row in miu], [o.pt_mul(o.G, x) for x in w], eks, proofs, S, c_a, c_bw)
    p7 = dict(s_vec=s_vec, r=r, R_dash_vec=[o.pt_mul(R, x) for x in k], m=m, R=R, S_vec=S)
    return p5, p6, p7, R, dict(sigma=sigma, nonces=nonces, dks=dks, c_bw=c_bw, nu_rnd=nu_rnd)


def _corruptions(p5, p6, p7):
    """(name, phase, mutated state, expected bad actors)"""
    out = []
    x = copy.deepcopy(p5); x.delta_vec[1] = (x.delta_vec[1] + 1) % Q; out.append(("delta of signer 1", 5, x, [1]))
    x = copy.deepcopy(p5); x.gamma_vec[2] = (x.gamma_vec[2] + 1) % Q; out.append(("gamma of signer 2 opened wrong", 5, x, [2]))
    x = copy.deepcopy(p5); x.k_vec[0] = (x.k_vec[0] + 1) % Q; out.append(("k of signer 0 opened wrong", 5, x, [0]))
    x = copy.deepcopy(p5); x.beta_tag_vec[1][0] += 1; out.append(("beta' drawn by signer 0 for Alice 1 opened wrong", 5, x, [0]))
    x = copy.deepcopy(p5); x.beta_randomness_vec[2][1] += 1; out.append(("beta randomness of signer 1 for Alice 2", 5, x, [1]))
    x = copy.deepcopy(p6); x.S_vec[1] = o.pt_add(x.S_vec[1], o.G); out.append(("S of signer 1", 6, x, [1]))
    x = copy.deepcopy(p6); x.miu_randomness_vec[2][0] += 1; out.append(("miu randomness of signer 2", 6, x, [2]))
    x = copy.deepcopy(p6); x.miu_vec[0][1] += 1; out.append(("miu of signer 0", 6, x, [0]))
    x = copy.deepcopy(p6); x.proof_vec[2] = o.ECDDHProof(x.proof_vec[2].a1, x.proof_vec[2].a2, (x.proof_vec[2].z + 1) % Q); out.append(("ECDDH response of signer 2", 6, x, [2]))
    x = copy.deepcopy(p7); x["s_vec"][2] = (x["s_vec"][2] + 1) % Q; out.append(("s of signer 2", 7, x, [2]))
    x = copy.deepcopy(p7); x["S_vec"][0] = o.pt_add(x["S_vec"][0], o.G); out.append(("S of signer 0 in phase 7", 7, x, [0]))
    return out


def _run_oracle(phase, st, R):
    if phase == 5:
        return bo.phase5_blame(st)
    if phase == 6:
        return bo.phase6_blame(st, R)
    return bo.phase7_blame(**st)


def test_blame_oracle_finds_the_corrupted_signer(keyset):
    p5, p6, p7, R, extra = _transcript(keyset)
    assert bo.phase5_blame(p5) == [] and bo.phase6_blame(p6, R) == [] and bo.phase7_blame(**p7) == []
    # `Paillier::open` really inverts the encryption: the extracted randomness of Bob's MtAwc ciphertexts re-encrypts to them
    for i in range(3):
        for j in range(2):
            m, r = o.paillier_open(extra["dks"][i], extra["c_bw"][i][j])
            assert o.paillier_encrypt(p6.encryption_key_vec[i], m, r) == extra["c_bw"][i][j]
    for name, phase, st, want in _corruptions(p5, p6, p7):
        assert _run_oracle(phase, st, R) == want, name


def _pack_proofs(proofs):
    out = np.zeros((len(proofs), 40), np.uint32)
    for i, pf in enumerate(proofs):
        for off, p in ((0, pf.a1), (16, pf.a2)):
            out[i, off:off + 16] = np.frombuffer((p[0] | (p[1] << 256)).to_bytes(64, "little"), dtype="<u4")
        out[i, 32:40] = np.frombuffer(pf.z.to_bytes(32, "little"), dtype="<u4")
    return out


@pytest.mark.gpu
def test_blame_on_gpu_matches_oracle(engine, pkg, keyset):
    from mpecdsa_b200 import blame, gg20
    p5, p6, p7, R, extra = _transcript(keyset)
    ks = gg20.KeySets(engine, [keyset])
    n_list = [ek.n for ek in p5.encryption_key_vec]
    # new primitives first: Paillier::open and ECDDHProof, bit-exact
    cs = [extra["c_bw"][i][j] for i in range(3) for j in range(2)]
    m, r = blame.paillier_open(engine, ks, [i for i in range(3) for _ in range(2)], cs)
    assert list(zip(m, r)) == [o.paillier_open(extra["dks"][i], extra["c_bw"][i][j]) for i in range(3) for j in range(2)]
    G = o.G
    h1 = [o.pt_mul(G, s) for s in extra["sigma"]]
    got = blame.ecddh_prove(engine, extra["sigma"], [G] * 3, h1, [R] * 3, p6.S_vec, extra["nonces"])
    assert np.array_equal(got, _pack_proofs(p6.proof_vec))
    assert list(blame.ecddh_verify(engine, got, [G] * 3, h1, [R] * 3, p6.S_vec)) == [0, 0, 0]
    assert list(blame.ecddh_verify(engine, got, [G] * 3, h1, [R] * 3, [p6.S_vec[1], p6.S_vec[1], p6.S_vec[2]])) == [pkg.ST_PROOF, 0, 0]

    def run(phase, st):
        if phase == 5:
            return blame.phase5_blame(engine, n_list, st.k_vec, st.k_randomness_vec, st.gamma_vec, st.beta_randomness_vec, st.beta_tag_vec, st.delta_vec,
                                      st.g_gamma_vec, st.m_a_c, st.m_b_c)
        if phase == 6:
            return blame.phase6_blame(engine, n_list, st.k_vec, st.k_randomness_vec, st.miu_vec, st.miu_randomness_vec, st.g_w_vec, _pack_proofs(st.proof_vec),
                                      st.S_vec, st.m_a_c, st.m_b_c, R)
        return blame.phase7_blame(engine, st["s_vec"], st["r"], st["R_dash_vec"], st["m"], st["R"], st["S_vec"])

    assert run(5, p5) == [] and run(6, p6) == [] and run(7, p7) == []
    for name, phase, st, want in _corruptions(p5, p6, p7):
        assert run(phase, st) == _run_oracle(phase, st, R) == want, name
    ks.free()


@pytest.mark.gpu
@pytest.mark.parametrize("edge", [0, 1, 2], ids=lambda k: f"edge{k}")
def test_blame_on_gpu_matches_oracle_on_edge_keysets(engine, pkg, edge):
    """the same transcript and corruptions on each key set of keys_edge.json (2047-bit N, p < q, p/q close to 2 and to 4)"""
    test_blame_on_gpu_matches_oracle(engine, pkg, fixtures.load_edge_keysets()[edge])


@pytest.mark.gpu
def test_paillier_open_on_edge_rows(engine):
    """`Paillier::open` on every edge row: m = r = N - 1; c = N^2 - 1 (m = 0, r = N - 1); the plaintexts with (m mod p, m mod q) =
    (p - 1, 0) and (0, q - 1), whose CRT tail needs the most corrections; and c + k N^2 < 2^4096 with its high 2048-bit half above N,
    which a 2047-bit N allows: the job that computes r then reduces a high half larger than its modulus.  m and r equal the
    oracle's, and (1 + m N) r^N = c mod N^2."""
    from mpecdsa_b200 import blame, gg20
    rows = [lk for ks in fixtures.load_edge_keysets() for lk in ks]
    shapes = [r["shape"] for ks in fixtures.edge_keysets_raw() for r in ks["parties"]]
    rng = random.Random(0x09E4)
    idx, cs, kinds = [], [], []
    for i, lk in enumerate(rows):
        n = lk.dk.p * lk.dk.q
        ek = o.EncryptionKey(n, n * n)
        cases = [("m = r = N - 1", o.paillier_encrypt(ek, n - 1, n - 1)), ("N^2 - 1", ek.nn - 1)]
        cases += [("worst residues", o.paillier_encrypt(ek, m, n - 1)) for m in _worst_plaintexts(lk.dk.p, lk.dk.q)]
        c0 = o.paillier_encrypt(ek, rng.randrange(n), rng.randrange(1, n))
        wide = c0 + ((1 << 4096) - 1 - c0) // ek.nn * ek.nn
        assert wide >> 2048 > n or n.bit_length() == 2048, shapes[i]
        if wide >> 2048 > n:
            cases.append(("high half above N", wide))
        for kind, c in cases:
            idx.append(i); cs.append(c); kinds.append((shapes[i], kind))
    assert sum(k == "high half above N" for _, k in kinds) >= 5
    ks = gg20.KeySets(engine, fixtures.load_edge_keysets())
    try:
        m, r = blame.paillier_open(engine, ks, idx, cs)
    finally:
        ks.free()
    want = [o.paillier_open(rows[i].dk, c) for i, c in zip(idx, cs)]
    assert [kinds[j] for j in range(len(cs)) if (m[j], r[j]) != want[j]] == []
    for i, c, mm, rr in zip(idx, cs, m, r):
        n = rows[i].dk.p * rows[i].dk.q
        assert (1 + mm * n) * pow(rr, n, n * n) % (n * n) == c % (n * n)
