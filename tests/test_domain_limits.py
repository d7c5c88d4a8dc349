"""CPU tests at the edge of the declared domain of the one-call drivers (key sets of up to 64 parties, signing sets of up to all
of them, t up to n - 1, bad-actor masks with bits up to 63): the host-harness builds of the Lagrange, index, round-2 and MessageB
status kernels at T = 64 of P = 64 and for signing sets that contain party 64, the keygen finish kernel at n = 64 with failing
senders 33 and 64; and the plain scalar reference of the MtA shares that tests/test_domain_limits_gpu.py checks 64-signer
sessions with, itself checked here against the party-by-party oracles of GG20 and GG18 on small sessions."""
import dataclasses
import random

import numpy as np

from oracle import gg20_general_oracle as gen
from oracle import gg20_oracle as o
from tests import gg18_signing_oracle as so
from tests import keygen_group as kgg
from tests.golden import fixtures
from tests.test_gg20_keygen import _finish, hk  # noqa: F401  (hk is the module fixture of the keygen harness)
from tests.test_gg20_offline_general import I, L, P_, from16, hg, pt16, rows  # noqa: F401  (hg: the offline-stage harness)

Q, G = o.Q, o.G
OK, INVALID_KEY = 0, 2


def _ind(p, j):
    return j if j < p else j + 1


# ------------------------------------------------------------------------------------------------ the scalar reference
@dataclasses.dataclass
class MtaSession:
    mta_bad: list          # per position: a MessageB it received fails verify_proofs_get_alpha (alpha != k b + beta' mod q)
    key_bad: list          # per position: a peer's MessageB(w) carries a key other than lambda * pk_vec (rounds.rs:281)
    delta: list
    sigma: list
    R: object = None       # delta^-1 * sum gamma_j G, when no check failed
    T: list = None         # sigma_i G + l_i H, when no check failed


def mta_session(keys, l_s, k, gamma, bt_gamma, bt_w, l=None):
    """Round 0..2 of one signing session with plain integers, no Paillier: keys[p] the LocalKey of signer position p, l_s[p] its
    keygen index - 1, k / gamma / l per position, bt_gamma[b][j] / bt_w[b][j] the beta' that Bob b draws towards Alice ind(b, j).
    Alice a's share of (k_a, x_b) is the decryption of Enc(k_a)^x_b * Enc(beta') mod q, i.e. ((k_a x_b + beta') mod N_a) mod q, and
    Bob keeps -beta' mod q; the MessageB check (mta/mod.rs:160-179) holds iff no wrap mod N_a changed the share mod q."""
    T = len(l_s)
    k, gamma = [v % Q for v in k], [v % Q for v in gamma]
    w = [o.lagrange_at_zero(l_s[p], l_s) * keys[p].x_i % Q for p in range(T)]
    own_key = [o.pt_mul(G, keys[b].x_i) == keys[b].pk_vec[l_s[b]] for b in range(T)]
    delta = [k[p] * gamma[p] for p in range(T)]
    sigma = [k[p] * w[p] for p in range(T)]
    mta_bad, key_bad = [False] * T, [False] * T
    for a in range(T):
        N = keys[a].paillier_key_vec[l_s[a]].n
        for j in range(T - 1):
            b = _ind(a, j)
            jb = a if a < b else a - 1                              # Bob b's slot towards Alice a
            for x, bt, acc in ((gamma[b], bt_gamma[b][jb], delta), (w[b], bt_w[b][jb], sigma)):
                alpha = (k[a] * x + bt) % N % Q
                mta_bad[a] = mta_bad[a] or alpha != (k[a] * x + bt) % Q
                acc[a] += alpha
                acc[b] -= bt
            key_bad[a] = key_bad[a] or not own_key[b]
    res = MtaSession(mta_bad, key_bad, [d % Q for d in delta], [s % Q for s in sigma])
    if not any(mta_bad) and not any(key_bad):
        res.R = o.pt_mul(G, sum(gamma) * pow(sum(res.delta) % Q, -1, Q) % Q)
        if l is not None:
            res.T = [o.pt_add(o.pt_mul(G, res.sigma[p]), o.pt_mul(o.H2, l[p] % Q)) for p in range(T)]
    return res


def signature(ref, k, message):
    """the GG18 / GG20 online step on the reference shares: s_i = m k_i + r sigma_i, then (r, s, recid) with low s"""
    return o.output_signature(ref.R, [o.local_sig(k[p] % Q, message, ref.R, ref.sigma[p]) for p in range(len(k))])


# ------------------------------------------------------------------------------------------------ the reference against the oracles
def _keyset():
    return fixtures.load_keyset(0)


def test_scalar_reference_equals_gg20_oracle():
    """gen.offline_session and mta_session agree on R, sigma_i and T_i of complete sessions, and on who fails round 2 for a wrong
    x_i, a beta' of N_a - 1 (the share wraps mod N_a) and a beta' of -k_a gamma_b mod q (Alice's share is zero)"""
    from tests.test_gg20_general import _party_randomness
    keys = _keyset()
    rng = random.Random(0xD0A1)
    cases = [([3, 1, 2], None, ("gamma", "zero")), ([2, 3], "x", None), ([1, 3], None, ("gamma", "wrap")), ([3, 2], None, ("w", "wrap"))]
    for s_l, tamper, bt in cases:
        ks = [keys[i - 1] for i in s_l]
        if tamper:
            ks[1] = dataclasses.replace(ks[1], x_i=(ks[1].x_i + 1) % Q)
        rnd = [_party_randomness(rng, lk, [s_l[_ind(p, j)] - 1 for j in range(len(s_l) - 1)]) for p, lk in enumerate(ks)]
        if bt:
            a, b = 0, 1                                              # Bob 1 towards Alice 0 (slot 0)
            N = ks[a].paillier_key_vec[s_l[a] - 1].n
            zero = -(rnd[a].k_i % Q) * (rnd[b].gamma_i % Q) % Q
            getattr(rnd[b], "beta_tag_" + bt[0])[0] = N - 1 if bt[1] == "wrap" else zero
        want = gen.offline_session(ks, s_l, rnd)
        l_s = [i - 1 for i in s_l]
        ref = mta_session(ks, l_s, [r.k_i for r in rnd], [r.gamma_i for r in rnd], [r.beta_tag_gamma for r in rnd],
                          [r.beta_tag_w for r in rnd], [r.l for r in rnd])
        assert [r.status for r in want] == [INVALID_KEY if m or kb else OK for m, kb in zip(ref.mta_bad, ref.key_bad)], (s_l, tamper, bt)
        if tamper:
            assert ref.key_bad == [True, False] + [True] * (len(s_l) - 2)
        if bt:
            assert ref.mta_bad[0] == (bt[1] == "wrap") and not any(ref.mta_bad[1:])
        if all(r.status == OK for r in want):
            for p, r in enumerate(want):
                assert (r.R, r.sigma_i, r.t_vec) == (ref.R, ref.sigma[p], ref.T), (s_l, p)


def test_scalar_reference_equals_gg18_restatement():
    """so.sign_session and mta_session agree on R, sigma_i and the signature of a complete session, and on who fails for a
    wrapping beta'"""
    from tests.test_gg18_signing import random_signers
    keys = _keyset()
    rng = random.Random(0xD018)
    for s_l, wrap in (([2, 3, 1], False), ([1, 3], True)):
        ks = [keys[i - 1] for i in s_l]
        rnd = random_signers(ks, s_l, rng)
        if wrap:
            rnd[0].beta_tag_w[0] = ks[1].paillier_key_vec[s_l[1] - 1].n - 1           # Bob 0 towards Alice 1
        m = rng.getrandbits(256) % Q
        want = so.sign_session(ks, s_l, rnd, m)
        ref = mta_session(ks, [i - 1 for i in s_l], [r.k for r in rnd], [r.gamma for r in rnd], [r.beta_tag_gamma for r in rnd],
                          [r.beta_tag_w for r in rnd])
        if wrap:
            assert want.status == [OK, INVALID_KEY] and ref.mta_bad == [False, True]
            continue
        assert want.status == [OK] * 3 and not any(ref.mta_bad + ref.key_bad)
        assert want.sigma == ref.sigma and want.delta == ref.delta and want.R == [ref.R] * 3
        assert want.signature == signature(ref, [r.k for r in rnd], m)


# ------------------------------------------------------------------------------------------------ offline-stage kernels at T = 64
def test_lagrange_at_64_signers_and_party_64(hg):
    """w = lambda x_i and g_w = lambda pk for all 64 signers of a 64-party key set in two orders, and for small signing sets that
    contain party 64; the Lagrange-weighted shares of a degree-63 sharing sum to the secret"""
    rng = random.Random(0x640A)
    P = 64
    coef = [rng.randrange(1, Q) for _ in range(P)]
    f = lambda x: sum(c * pow(x, k, Q) for k, c in enumerate(coef)) % Q
    xi = [f(i + 1) for i in range(P)] + [rng.randrange(1, Q) for _ in range(P)]
    pk = [o.pt_mul(G, x) for x in xi]
    XI, PK = rows(xi, 8), np.stack([pt16(p) for p in pk])
    perm = list(range(P))
    rng.shuffle(perm)
    for d in ([[0] + list(range(P)), [1] + perm, [0] + perm[::-1]], [[0, 63, 0], [1, 0, 63], [1, 32, 63]], [[0, 31, 63, 32], [1, 63, 8, 9]]):
        T = len(d[0]) - 1
        E = len(d) * T
        w, gw = np.zeros((E, 8), np.uint32), np.zeros((E, 16), np.uint32)
        hg.h_lagrange(P_(np.array(d, np.uint32)), T, P, P_(XI), P_(PK), P_(w), P_(gw), E)
        for u in range(E):
            s, p = divmod(u, T)
            l_s = d[s][1:]
            lam = o.lagrange_at_zero(l_s[p], l_s)
            r = d[s][0] * P + l_s[p]
            assert I(w[u]) == lam * xi[r] % Q, (T, u)
            if T < P or u % 8 == 0:                                     # a sample of the 192 point products at T = 64
                assert from16(gw[u]) == o.pt_mul(pk[r], lam), (T, u)
        if T == P:
            assert sum(I(w[p]) for p in range(T)) % Q == coef[0]
            assert sum(I(w[2 * T + p]) for p in range(T)) % Q == coef[0]


def test_pair_tables_round_trip_at_64(hg):
    """k_gen_index at T = P = 64: every pair's receiving element and key row follow peer_of, and the pair that answers it
    (pair_to) leads back to the sender"""
    rng = random.Random(0x640B)
    T = P = 64
    d = [[0] + list(range(P)), [1] + rng.sample(range(P), P)]
    E, NP = 2 * T, (T - 1) * 2 * T
    out = [np.zeros(x, np.uint32) for x in (E, P * E, P * E, 2 * NP, 2 * NP, 2 * NP)]
    hg.h_index(P_(np.array(d, np.uint32)), T, P, E, *[P_(a) for a in out])
    row, st_row, st_elem, me, peer, row_peer = out
    own = [d[u // T][0] * P + d[u // T][1 + u % T] for u in range(E)]
    assert list(row) == own
    assert list(st_row) == [d[t % E // T][0] * P + t // E for t in range(P * E)] and list(st_elem) == [t % E for t in range(P * E)]
    for t in range(2 * NP):
        q = t % NP
        u, j = q % E, q // E
        v = u - u % T + _ind(u % T, j)
        assert (me[t], peer[t], row_peer[t]) == (u, v, own[v])
        pu, pv = u % T, v % T
        back = (pu if pu < pv else pu - 1) * E + v                     # pair_to(T, E, v, u)
        assert (me[back], peer[back]) == (v, u)


def test_round2_and_msgb_status_at_64(hg):
    """delta_i and sigma_i over 63 incoming and 63 outgoing pairs per element, the MessageB(w) key check against a distinct g_w per
    sender, and the MessageB status of a failed range proof at statement 63"""
    rng = random.Random(0x640C)
    T = 64
    E, NP = T, (T - 1) * T
    pair = lambda b, v: ((v % T) if (v % T) < (b % T) else (v % T) - 1) * E + b           # b sends to v
    k, gam, w = ([rng.randrange(1, Q) for _ in range(E)] for _ in range(3))
    gw_s = [rng.randrange(1, Q) for _ in range(E)]
    gw = [o.pt_mul(G, x) for x in gw_s]
    alpha = [rng.randrange(Q) for _ in range(2 * NP)]
    beta = [rng.randrange(Q) for _ in range(2 * NP)]
    bp = np.zeros((2 * NP, 40), np.uint32)
    for b in range(E):
        for v in range(E):
            if v != b:
                bp[NP + pair(b, v), :16] = pt16(gw[b])
    bp[NP + pair(40, 50), :16] = pt16(gw[41])                      # 41's key in the MessageB(w) element 40 sends element 50
    st_a = np.zeros(2 * NP, np.uint8)
    st_a[pair(63, 33)] = INVALID_KEY                                # element 33 fails get_alpha on what element 63 sent it
    delta, sigma, cand = np.zeros((E, 8), np.uint32), np.zeros((E, 8), np.uint32), np.zeros(E, np.uint8)
    args = [rows(alpha, 8), rows(beta, 8), bp, np.stack([pt16(p) for p in gw]), rows(k, 8), rows(gam, 8), rows(w, 8)]
    hg.h_round2(T, E, P_(st_a), *[P_(a) for a in args], P_(delta), P_(sigma), P_(cand))
    for v in range(E):
        ins = [pair(b, v) for b in range(E) if b != v]
        outs = [j * E + v for j in range(T - 1)]
        assert I(delta[v]) == (k[v] * gam[v] + sum(alpha[t] for t in ins) + sum(beta[t] for t in outs)) % Q, v
        assert I(sigma[v]) == (k[v] * w[v] + sum(alpha[NP + t] for t in ins) + sum(beta[NP + t] for t in outs)) % Q, v
    assert [u for u in range(E) if cand[u]] == [33, 50] and set(cand[[33, 50]]) == {INVALID_KEY}
    # one failed range proof (statement 63 of element 40's MessageA) fails every MessageB that answers element 40
    P = 64
    pst = np.zeros(P * E, np.uint8)
    pst[63 * E + 40] = 5
    pair_st = np.full(2 * NP, 255, np.uint8)
    hg.h_msgb_status(P_(pst), P, T, E, P_(pair_st), NP)
    for t in range(2 * NP):
        q = t % NP
        assert pair_st[t] == (5 if _ind(q % E, q // E) == 40 else 0), t


# ------------------------------------------------------------------------------------------------ keygen finish at n = 64
def test_keygen_finish_masks_at_64(hk):
    """k_kg_finish for two groups of 64: the failing senders 33 and 64 give the mask 2^32 + 2^63 as that exact integer, in every
    round that names senders; the first failing round decides; the other group completes untouched"""
    n = t1 = 64
    E = 2 * n
    high = (1 << 32) | (1 << 63)
    ones = np.ones(E, np.uint8)
    pair = np.ones(E * n, np.uint8)
    fail2, fail4 = ones.copy(), ones.copy()
    fail2[[32, 63]] = 0
    fail4[[32, 63]] = 0
    fail3 = pair.copy()
    fail3[0 * n + 63] = 0                                           # receiver 1 rejects sender 64's share
    fail3[63 * n + 32] = 0                                          # receiver 64 rejects sender 33's share
    fail3[40 * n + 32] = 0
    fail3[40 * n + 63] = 0                                          # receiver 41 rejects both
    st_nt = np.zeros(E, np.uint8)
    # round 2 alone, then with later failures too: every element of group 0 INVALID_KEY with both senders
    for p3, p4 in ((pair, ones), (fail3, fail4)):
        out, proof, gcomm = _finish(hk, n, t1, st_nt, fail2, p3, p4)
        assert [int(b) for b in out["bad"][:n]] == [high] * n and list(out["status"][:n]) == [kgg.ST_INVALID_KEY] * n
        assert list(out["complete"]) == [0, 1] and list(out["status"][n:]) == [0] * n and not out["bad"][n:].any()
        assert not out["pk"][:n].any() and (out["pk"][n:] == proof[n:, :16]).all() and (out["y"][1] == gcomm[1, 0]).all()
    # round 3: each receiver names its own failing senders
    out, _, _ = _finish(hk, n, t1, st_nt, ones, fail3, fail4)
    want = [0] * n
    want[0], want[63], want[40] = 1 << 63, 1 << 32, high
    assert [int(b) for b in out["bad"][:n]] == want
    assert list(out["status"][:n]) == [kgg.ST_INVALID_SS if m else 0 for m in want] and out["complete"][0] == 0
    # round 4
    out, _, _ = _finish(hk, n, t1, st_nt, ones, pair, fail4)
    assert [int(b) for b in out["bad"][:n]] == [high] * n and list(out["status"][:n]) == [kgg.ST_PROOF] * n
    # round 0 comes first: an uninvertible xhi at party 64 hides every later failure
    st_nt[63] = kgg.ST_NOT_INVERTIBLE
    out, _, _ = _finish(hk, n, t1, st_nt, fail2, fail3, fail4)
    assert list(out["status"][:n]) == [0] * 63 + [kgg.ST_NOT_INVERTIBLE] and not out["bad"].any() and list(out["complete"]) == [0, 1]
