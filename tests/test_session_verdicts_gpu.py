"""The fused GG20 offline stage with each Pedersen, PDL-with-slack and HomoElGamal proof of a session verified once, on its
prover's unit (declared shortcut 10, DESIGN.md section 4), against the C twin of the oracle (oracle/gg20_twin.c), which runs
every check on both units:

- the non-invertible ciphertext records of test_kernel_variants_gpu (the round-1 and round-5 invertibility flags) and the edge
  keys of tests/golden/keys_edge.json: statuses, R, sigma_i, t_vec and the transcript digest bit for bit;
- records with k_i = 0 and with the PDL alpha = 0 or a multiple of q, which the oracle refuses (the reference panics on the
  point at infinity they produce): R is still bit-identical on both units of those sessions, and the other sessions of the
  same batch equal the twin;
- the six arena fields of the removed second checks are gone from tecdsa_gg20_debug_field;
- the multiply-accumulates the kernels count per unit fall by at least 45 M against the parent commit's job lists."""
import os

import numpy as np
import pytest

from oracle.sampling import Drbg, sample_unit
from tests.golden import fixtures

pytestmark = pytest.mark.gpu

_Q = 0xFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFEBAAEDCE6AF48A03BBFD25E8CD0364141
PAIRS = [(0, 1), (0, 2), (1, 2), (1, 0), (2, 0), (2, 1)]
REMOVED = ("VE1", "VLIN1", "VZE1", "VZEI1", "VU21", "VU31")
# executed MAC32 per unit of the work batch below (256 sessions over the 8 standard key sets, synthetic_batch seed 0x5E55),
# counted by the kernels (tecdsa_ctx_work) at the parent commit, where every unit also checked its peer's proofs
PARENT_MAC32_PER_UNIT = 451_004_920


def _twin(keysets, sess, rnd):
    from oracle import twin
    return twin.offline_batch(twin.KeyTables(keysets), np.asarray(sess, np.uint32), rnd, os.cpu_count() or 1)


def _assert_matches_twin(res, tw, sessions):
    """a session the twin completes is bit-equal to it on every output; in a session the twin stops, the unit the twin rejects
    has the twin's status and its peer is not reported OK (the batch runs every round, so the peer fails a later check)"""
    for s in sessions:
        u = slice(2 * s, 2 * s + 2)
        if tw.status[u].any():
            for v in (2 * s, 2 * s + 1):
                assert res.status[v] == tw.status[v] if tw.status[v] else res.status[v] != 0, (s, list(res.status[u]), list(tw.status[u]))
            continue
        assert not res.status[u].any(), (s, list(res.status[u]))
        for f in ("R", "sigma", "t_vec", "digest"):
            assert np.array_equal(getattr(res, f)[u], getattr(tw, f)[u]), (s, f)


def test_noninvertible_ciphertext_records_match_twin(engine, pkg, keyset):
    """the round-5 invertibility flag of the prover's own ciphertext (byte 8) stands in for the verifier's round-1 flag of the
    same ciphertext (byte 3); the Kaliski fallback of the inverses runs the same records in
    test_kernel_variants_gpu::test_kernel_variant_matches_oracle_and_default[kaliski]"""
    from mpecdsa_b200 import gg20
    from tests.test_kernel_variants_gpu import _inverse_session_inputs
    sess, rnds, _ = _inverse_session_inputs(keyset)
    rnd = gg20.pack_randomness(rnds)
    ks = gg20.KeySets(engine, [keyset])
    try:
        res = gg20.offline_batch(engine, ks, sess, rnd)
    finally:
        ks.free()
    tw = _twin([keyset], sess, rnd)
    assert list(tw.status) == [pkg.ST_INVALID_KEY, 0, 0, pkg.ST_INVALID_KEY, pkg.ST_INVALID_KEY, 0, 0, 0, 0, 0]
    _assert_matches_twin(res, tw, range(len(sess)))
    for s in range(len(sess)):
        assert np.array_equal(res.R[2 * s], res.R[2 * s + 1]), s


def test_edge_keys_match_twin(engine, pkg):
    from mpecdsa_b200 import gg20
    edge = fixtures.load_edge_keysets()
    rng = Drbg(0x5E56, "session-verdicts-edge")
    sess, rnds = [], []
    for k, ks_ in enumerate(edge):
        for a, b in PAIRS:
            keys, s_l = [ks_[a], ks_[b]], [a + 1, b + 1]
            rnds += [sample_unit(rng, keys, s_l, p) for p in range(2)]
            sess.append((k, a, b))
    rnd = gg20.pack_randomness(rnds)
    ks = gg20.KeySets(engine, edge)
    try:
        res = gg20.offline_batch(engine, ks, sess, rnd)
    finally:
        ks.free()
    tw = _twin(edge, sess, rnd)
    assert not tw.status.any() and not res.status.any()
    _assert_matches_twin(res, tw, range(len(sess)))


def test_R_identical_on_both_units_with_k_zero_and_alpha_zero(engine, keyset):
    """k_i = 0 puts R_dash at infinity and alpha = 0 mod q the PDL u1; both leave their unit's R untouched, so both units of
    the session hold the same R and read the same proof verdicts"""
    from mpecdsa_b200 import gg20
    rng = Drbg(0x5E57, "session-verdicts-zero")
    sess, rnds = [], []
    for a, b in PAIRS:
        keys, s_l = [keyset[a], keyset[b]], [a + 1, b + 1]
        rnds += [sample_unit(rng, keys, s_l, p) for p in range(2)]
        sess.append((0, a, b))
    rnds[0].k_i = 0                                                   # session 0: k = 0 on its first unit
    rnds[3].pdl = (0,) + tuple(rnds[3].pdl[1:])                       # session 1: alpha = 0 on its second unit
    rnds[4].pdl = (_Q,) + tuple(rnds[4].pdl[1:])                      # session 2: alpha = q, and k = 0 on the peer
    rnds[5].k_i = 0
    special = {0, 1, 2}
    rnd = gg20.pack_randomness(rnds)
    ks = gg20.KeySets(engine, [keyset])
    try:
        res = gg20.offline_batch(engine, ks, sess, rnd)
    finally:
        ks.free()
    for s in range(len(sess)):
        assert np.array_equal(res.R[2 * s], res.R[2 * s + 1]), s
    keep = [s for s in range(len(sess)) if s not in special]
    idx = [u for s in keep for u in (2 * s, 2 * s + 1)]
    tw = _twin([keyset], [sess[s] for s in keep], rnd[idx])

    class Sub:
        pass
    sub = Sub()
    for f in ("status", "R", "sigma", "t_vec", "digest"):
        setattr(sub, f, getattr(res, f)[idx])
    assert not tw.status.any()
    _assert_matches_twin(sub, tw, range(len(keep)))


def test_debug_field_refuses_the_removed_fields(engine, pkg, keyset):
    from mpecdsa_b200 import gg20
    rng = Drbg(0x5E58, "session-verdicts-debug")
    keys, s_l = [keyset[0], keyset[1]], [1, 2]
    rnd = gg20.pack_randomness([sample_unit(rng, keys, s_l, p) for p in range(2)])
    ks = gg20.KeySets(engine, [keyset])
    try:
        gg20.offline_batch(engine, ks, [(0, 0, 1)], rnd)
    finally:
        ks.free()
    for name in REMOVED:
        with pytest.raises(pkg.EngineError, match="unknown field"):
            gg20.debug_field(engine, name, 2)
    for name in ("VE0", "VLIN0", "VZE0", "VZEI0", "VCEI0", "VU20", "VU30"):
        assert gg20.debug_field(engine, name, 2).any(), name


def test_counted_work_drops_by_the_removed_checks(engine):
    from mpecdsa_b200 import gg20
    keysets = fixtures.load_all_keysets()
    sess, rnd = gg20.synthetic_batch(keysets, 256, 0x5E55)
    ks = gg20.KeySets(engine, keysets)
    try:
        engine.work(reset=True)
        res = gg20.offline_batch(engine, ks, sess, rnd)
        per_unit = engine.work() / (2 * len(sess))
    finally:
        ks.free()
    assert not res.status.any()
    assert per_unit <= PARENT_MAC32_PER_UNIT - 45e6, per_unit
