"""The GG20 offline stage for signing sets other than the two-of-three work unit: the size-generic oracle against the two-party
oracle (CPU), and the driver that runs any signing set as batch calls of the C ABI against the size-generic oracle (GPU) — the
reference's own integration tests run (t, n, signers) = (1, 3, [1,2]), (2, 3, [1,2,3]) and larger
(/root/reference/src/protocols/multi_party_ecdsa/gg_2020/state_machine/sign.rs:728-760)."""
import random

import numpy as np
import pytest

from oracle import gg20_general_oracle as gen
from oracle import gg20_oracle as o

Q, G = o.Q, o.G


def _party_randomness(rng, lk, peer_keygen_indices):
    own = lk.i - 1
    n_own = lk.paillier_key_vec[own].n
    r = gen.PartyRandomness(gamma_i=rng.randrange(1, Q), k_i=rng.randrange(1, Q), blind=rng.getrandbits(256), r_k=rng.randrange(1, n_own))
    r.alice = [(rng.randrange(Q ** 3), rng.randrange(1, n_own), rng.randrange(Q ** 3 * st.N), rng.randrange(Q * st.N)) for st in lk.h1_h2_n_tilde_vec]
    for a in peer_keygen_indices:
        n_a = lk.paillier_key_vec[a].n
        st = lk.h1_h2_n_tilde_vec[a]
        r.beta_tag_gamma.append(rng.randrange(n_a)); r.r_gamma.append(rng.randrange(1, n_a))
        r.nonce_gamma_b.append(rng.randrange(1, Q)); r.nonce_gamma_beta.append(rng.randrange(1, Q))
        r.beta_tag_w.append(rng.randrange(n_a)); r.r_w.append(rng.randrange(1, n_a))
        r.nonce_w_b.append(rng.randrange(1, Q)); r.nonce_w_beta.append(rng.randrange(1, Q))
        r.pdl.append((rng.randrange(Q ** 3), rng.randrange(1, n_own), rng.randrange(Q * st.N), rng.randrange(Q ** 3 * st.N)))
    r.l, r.ped_s1, r.ped_s2, r.heg_s1, r.heg_s2 = (rng.randrange(1, Q) for _ in range(5))
    return r


def _session(rng, keyset, s_l):
    keys = [keyset[i - 1] for i in s_l]
    rnd = [_party_randomness(rng, lk, [s_l[gen._ind(p, j)] - 1 for j in range(len(s_l) - 1)]) for p, lk in enumerate(keys)]
    return keys, rnd


def _two_party_view(r):
    return o.UnitRandomness(gamma_i=r.gamma_i, k_i=r.k_i, blind=r.blind, r_k=r.r_k, alice=r.alice, beta_tag_gamma=r.beta_tag_gamma[0], r_gamma=r.r_gamma[0],
                            nonce_gamma_b=r.nonce_gamma_b[0], nonce_gamma_beta=r.nonce_gamma_beta[0], beta_tag_w=r.beta_tag_w[0], r_w=r.r_w[0],
                            nonce_w_b=r.nonce_w_b[0], nonce_w_beta=r.nonce_w_beta[0], l=r.l, ped_s1=r.ped_s1, ped_s2=r.ped_s2, pdl=r.pdl[0],
                            heg_s1=r.heg_s1, heg_s2=r.heg_s2)


def _signature_ok(res, y, rng):
    m = rng.getrandbits(256)
    r_, s_, _ = o.output_signature(res[0].R, [o.local_sig(x.k_i, m, x.R, x.sigma_i) for x in res])
    return o.ecdsa_verify(r_, s_, y, m)


def test_general_oracle_equals_two_party_oracle(keyset):
    rng = random.Random(0x6E1)
    s_l = [3, 1]
    keys, rnd = _session(rng, keyset, s_l)
    res = gen.offline_session(keys, s_l, rnd)
    two = o.offline_session(keys, s_l, [_two_party_view(r) for r in rnd])
    assert [(x.status, x.R, x.sigma_i, x.k_i, x.t_vec) for x in res] == [(x.status, x.R, x.sigma_i, x.k_i, x.t_vec) for x in two]
    assert all(x.status == 0 for x in res) and _signature_ok(res, keyset[0].y_sum_s, rng)


def test_general_oracle_three_signers(keyset):
    rng = random.Random(0x6E3)
    s_l = [2, 3, 1]
    keys, rnd = _session(rng, keyset, s_l)
    res = gen.offline_session(keys, s_l, rnd)
    assert [x.status for x in res] == [0, 0, 0] and all(x.R == res[0].R for x in res)
    assert _signature_ok(res, keyset[0].y_sum_s, rng)
    # signer position 1 runs with a wrong share: its MessageB(w) proof key is not g_w_vec[1], which every OTHER signer catches in
    # round 2 (the assert_eq! of rounds.rs:281, mapped to InvalidKey)
    import dataclasses
    bad_keys = list(keys)
    bad_keys[1] = dataclasses.replace(keys[1], x_i=(keys[1].x_i + 1) % Q)
    assert [x.status for x in gen.offline_session(bad_keys, s_l, rnd)] == [gen.ST_INVALID_KEY, 0, gen.ST_INVALID_KEY]


def _five_party_key(keysets, rng):
    """A (t = 2, n = 5) key over the Paillier keys / N~ setups of the fixture rows 0..4: fresh degree-2 Shamir sharing"""
    rows = [lk for ks in keysets for lk in ks][:5]
    coef = [rng.randrange(1, Q) for _ in range(3)]
    f = lambda x: (coef[0] + coef[1] * x + coef[2] * x * x) % Q
    x = [f(i + 1) for i in range(5)]
    y = o.pt_mul(G, coef[0])
    eks = [o.EncryptionKey(lk.dk.p * lk.dk.q, (lk.dk.p * lk.dk.q) ** 2) for lk in rows]
    sts = [lk.h1_h2_n_tilde_vec[lk.i - 1] for lk in rows]
    pks = [o.pt_mul(G, xi) for xi in x]
    return [o.LocalKey(i=i + 1, t=2, n=5, x_i=x[i], dk=rows[i].dk, pk_vec=pks, paillier_key_vec=eks, h1_h2_n_tilde_vec=sts, y_sum_s=y) for i in range(5)]


def _flatten(sessions, row_of):
    """sessions: list of (keys, s_l, rnd) with equal len(s_l) -> the driver's flat arguments"""
    ttag = len(sessions[0][1])
    key_rows, all_rows, w, g_w, y = [], [], [], [], []
    per_elem = {f: [] for f in ("gamma", "k", "blind", "r_k", "l", "ped_s1", "ped_s2", "heg_s1", "heg_s2", "alice")}
    per_pair = {f: [] for f in ("beta_tag_gamma", "r_gamma", "nonce_gamma_b", "nonce_gamma_beta", "beta_tag_w", "r_w", "nonce_w_b", "nonce_w_beta", "pdl")}
    for keys, s_l, rnd in sessions:
        l_s = [i - 1 for i in s_l]
        for p, (lk, r) in enumerate(zip(keys, rnd)):
            key_rows.append(row_of(lk, lk.i - 1))
            all_rows.append([row_of(lk, j) for j in range(lk.n)])
            lam = o.lagrange_at_zero(l_s[p], l_s)
            w.append(lam * lk.x_i % Q); g_w.append(o.pt_mul(lk.pk_vec[l_s[p]], lam)); y.append(lk.y_sum_s)
            for f, v in (("gamma", r.gamma_i), ("k", r.k_i), ("blind", r.blind), ("r_k", r.r_k), ("l", r.l), ("ped_s1", r.ped_s1), ("ped_s2", r.ped_s2),
                         ("heg_s1", r.heg_s1), ("heg_s2", r.heg_s2), ("alice", list(r.alice))):
                per_elem[f].append(v)
            for j in range(ttag - 1):
                for f in per_pair:
                    per_pair[f].append(getattr(r, f)[j])
    return ttag, key_rows, all_rows, w, g_w, y, {**per_elem, **per_pair}


def _check_messages(out, sessions):
    """the `Msg<OfflineProtocolMessage>` documents of every element: count, routing, and the fields the oracle can re-derive"""
    from mpecdsa_b200 import wire
    E = wire.DEFAULT
    u = 0
    for keys, s_l, rnd in sessions:
        ttag = len(s_l)
        for p, (lk, r) in enumerate(zip(keys, rnd)):
            msgs = out["messages"][u]
            assert [list(m["body"])[0] for m in msgs] == ["M1"] + ["M2"] * (ttag - 1) + ["M3", "M4", "M5", "M6"]
            assert all(m["sender"] == p + 1 for m in msgs)
            assert [m["receiver"] for m in msgs] == [None] + [gen._ind(p, j) + 1 for j in range(ttag - 1)] + [None] * 4
            m_a = o.message_a(r.k_i % Q, lk.paillier_key_vec[lk.i - 1], r.r_k, lk.h1_h2_n_tilde_vec, r.alice)
            want_a = wire.message_a(m_a.c, [{"z": x.z, "e": x.e, "s": x.s, "s1": x.s1, "s2": x.s2} for x in m_a.range_proofs])
            m1 = msgs[0]["body"]["M1"]
            assert m1[0] == want_a and m1[1] == wire.sign_broadcast_phase1(o.hash_commitment(o.bn_from_bytes(o.pt_compress(o.pt_mul(G, r.gamma_i % Q))), r.blind))
            m4 = msgs[ttag + 1]["body"]["M4"]
            assert m4 == wire.sign_decommit_phase1(r.blind, o.pt_mul(G, r.gamma_i % Q))
            m3 = msgs[ttag]["body"]["M3"]
            assert m3[1] == E.point(out["T"][u]) and m3[2]["com"] == m3[1] and set(m3[2]) == {"e", "a1", "a2", "com", "z1", "z2"}
            m5 = msgs[ttag + 2]["body"]["M5"]
            assert m5[0] == E.point(o.pt_mul(out["R"][u], out["k"][u])) and len(m5[1]) == ttag - 1 and set(m5[1][0]) == {"z", "u1", "u2", "u3", "s1", "s2", "s3"}
            m6 = msgs[ttag + 3]["body"]["M6"]
            assert m6[0] == E.point(o.pt_mul(out["R"][u], out["sigma"][u])) and set(m6[1]) == {"T", "A3", "z1", "z2"}
            u += 1


@pytest.mark.gpu
def test_general_signing_sets_on_gpu_match_oracle(engine, pkg):
    from mpecdsa_b200 import gg20, gg20_general
    from tests.golden import fixtures
    keysets = fixtures.load_all_keysets()[:2]
    ks = gg20.KeySets(engine, keysets)
    rng = random.Random(0x6E20)
    cases = []
    # (t = 1, n = 3): two and three signers, both key sets, permuted positions; fixture key set k occupies key rows 3k .. 3k+2
    for lists in ([(0, [1, 2]), (1, [3, 1]), (0, [2, 3])], [(0, [1, 2, 3]), (1, [3, 1, 2])]):
        sessions, owner = [], {}
        for kidx, s_l in lists:
            keys, rnd = _session(rng, keysets[kidx], s_l)
            sessions.append((keys, s_l, rnd))
            owner.update({id(lk): kidx for lk in keys})
        cases.append((sessions, owner))
    for sessions, owner in cases:
        out = gg20_general.offline_batch(engine, ks, *_flatten(sessions, lambda lk, j: 3 * owner[id(lk)] + j), messages=True)
        _check_messages(out, sessions)
        u = 0
        for keys, s_l, rnd in sessions:
            want = gen.offline_session(keys, s_l, rnd)
            for p, wv in enumerate(want):
                assert int(out["status"][u]) == wv.status == 0
                assert (out["R"][u], out["sigma"][u], out["k"][u], out["T"][u]) == (wv.R, wv.sigma_i, wv.k_i, wv.t_vec[p])
                u += 1
    # a failing party: signer 0 of the first two-signer session answers with a wrong w (MessageB proof key != g_w) -> its peer
    # stops with InvalidKey in round 2 (rounds.rs:281) and nothing is produced for the session; the other sessions are untouched
    sessions, owner = cases[0]
    args = list(_flatten(sessions, lambda lk, j: 3 * owner[id(lk)] + j))
    args[3] = list(args[3]); args[3][0] = (args[3][0] + 1) % Q
    out = gg20_general.offline_batch(engine, ks, *args)
    assert list(out["status"][:2]) == [0, pkg.ST_INVALID_KEY] and out["R"][0] is None and out["R"][1] is None
    assert list(out["status"][2:]) == [0] * (len(out["status"]) - 2) and all(r is not None for r in out["R"][2:])
    ks.free()
    # (t = 2, n = 5): three of five signers over fixture rows 0..4
    key5 = _five_party_key(keysets, rng)
    ks5 = gg20.KeySets(engine, keysets)
    s_l = [5, 2, 3]
    keys = [key5[i - 1] for i in s_l]
    rnd = [_party_randomness(rng, lk, [s_l[gen._ind(p, j)] - 1 for j in range(2)]) for p, lk in enumerate(keys)]
    want = gen.offline_session(keys, s_l, rnd)
    assert [x.status for x in want] == [0, 0, 0] and _signature_ok(want, key5[0].y_sum_s, rng)
    args = _flatten([(keys, s_l, rnd)], lambda lk, j: j)
    out = gg20_general.offline_batch(engine, ks5, *args)
    for p, wv in enumerate(want):
        assert int(out["status"][p]) == 0 and (out["R"][p], out["sigma"][p], out["k"][p], out["T"][p]) == (wv.R, wv.sigma_i, wv.k_i, wv.t_vec[p])
    ks5.free()


@pytest.mark.gpu
def test_general_signing_sets_on_edge_keys_match_oracle(engine):
    """The size-generic driver over keys_edge.json.  One batch holds a three-signer session on each edge key set, so 2047- and
    2048-bit moduli sit side by side and ciphertext and plaintext widths differ between the rows of every call; then a (t = 2, n = 5)
    key over edge rows 0..4, signed by three of them with both rows whose p/q is close to 4.  Every output equals the oracle's."""
    from mpecdsa_b200 import gg20, gg20_general
    from tests.golden import fixtures
    edge = fixtures.load_edge_keysets()
    ks = gg20.KeySets(engine, edge)
    rng = random.Random(0x6E2E)
    sessions, owner = [], {}
    for kidx, s_l in ((0, [2, 3, 1]), (1, [1, 2, 3]), (2, [3, 1, 2])):
        keys, rnd = _session(rng, edge[kidx], s_l)
        sessions.append((keys, s_l, rnd))
        owner.update({id(lk): kidx for lk in keys})
    try:
        out = gg20_general.offline_batch(engine, ks, *_flatten(sessions, lambda lk, j: 3 * owner[id(lk)] + j))
    finally:
        ks.free()
    u = 0
    for keys, s_l, rnd in sessions:
        want = gen.offline_session(keys, s_l, rnd)
        assert _signature_ok(want, keys[0].y_sum_s, rng)
        for p, wv in enumerate(want):
            assert int(out["status"][u]) == wv.status == 0
            assert (out["R"][u], out["sigma"][u], out["k"][u], out["T"][u]) == (wv.R, wv.sigma_i, wv.k_i, wv.t_vec[p]), (s_l, p)
            u += 1
    key5 = _five_party_key(edge, rng)
    s_l = [5, 1, 3]                                   # edge rows 4 (q/p ~ 4), 0 (p/q ~ 4) and 2 (N just below 2^2048)
    assert [(lk.dk.p * lk.dk.q).bit_length() for lk in (key5[i - 1] for i in s_l)] == [2047, 2047, 2048]
    keys = [key5[i - 1] for i in s_l]
    rnd = [_party_randomness(rng, lk, [s_l[gen._ind(p, j)] - 1 for j in range(2)]) for p, lk in enumerate(keys)]
    want = gen.offline_session(keys, s_l, rnd)
    assert [x.status for x in want] == [0, 0, 0] and _signature_ok(want, key5[0].y_sum_s, rng)
    ks5 = gg20.KeySets(engine, edge)
    try:
        out = gg20_general.offline_batch(engine, ks5, *_flatten([(keys, s_l, rnd)], lambda lk, j: j))
    finally:
        ks5.free()
    for p, wv in enumerate(want):
        assert int(out["status"][p]) == 0 and (out["R"][p], out["sigma"][p], out["k"][p], out["T"][p]) == (wv.R, wv.sigma_i, wv.k_i, wv.t_vec[p])
