"""Round 1's AliceProof u' of the fused GG20 offline stage evaluated through the CRT halves of the peer's key row (declared
shortcut 12, DESIGN.md section 4): s^N runs as a 1024-bit stage and a p-adic stage whose Straus job also carries (c^-1)^e as
its second base and (s1 N + 1) as its multiplier, the first two-base jobs of the p^2 / q^2 kernel.

- A batch over a standard and the three edge key sets in which every prover draws r_k and the range proofs' beta from
  {0, 1, p, q, N - 1} of its own key, so that the verifier's s = r^e * beta mod N_peer is 0, 1, a multiple of p or of q, or
  N - 1, and some ciphertexts are not units mod N^2: UV0..UV2 equal the Python value of every unit, and status, R, sigma_i,
  t_vec and digest equal the C twin of the oracle.
- The counted work per unit falls by at least 60 M MAC32 against the parent commit, where the three u' ran as N-adic jobs,
  and the p-adic job list has one launch more per call while the N^2 list keeps its five."""
import numpy as np
import pytest

from oracle.sampling import Drbg, sample_unit
from tests.golden import fixtures
from tests.test_session_verdicts_gpu import PAIRS, _assert_matches_twin, _twin

pytestmark = pytest.mark.gpu

# executed MAC32 per unit of synthetic_batch(load_all_keysets(), 256, 0x5E55), counted by the kernels (tecdsa_ctx_work) at
# the parent commit, and that commit's launches of the p-adic job list per offline call
PARENT_MAC32_PER_UNIT = 401_471_653
PARENT_PADIC_LAUNCHES = 4


def _int(row):
    return int.from_bytes(np.ascontiguousarray(row).tobytes(), "little")


def test_peer_u_prime_at_special_witnesses(engine, pkg):
    from mpecdsa_b200 import gg20
    keysets = [fixtures.load_keyset(0)] + fixtures.load_edge_keysets()
    rng = Drbg(0x9EE2, "peer-crt")
    sess, rnds, peer_keys = [], [], []
    j = 0
    for k, ks_ in enumerate(keysets):
        for a, b in PAIRS:
            keys, s_l = [ks_[a], ks_[b]], [a + 1, b + 1]
            for pos in range(2):
                r = sample_unit(rng, keys, s_l, pos)
                dk = keys[pos].dk
                pick = (0, 1, dk.p, dk.q, dk.p * dk.q - 1)
                r.r_k = pick[j % 5]
                r.alice = [(al, pick[(j // 5 + x) % 5]) + tuple(rest) for x, (al, _, *rest) in enumerate(r.alice)]
                rnds.append(r)
                peer_keys.append(keys[1 - pos].dk)
                j += 1
            sess.append((k, a, b))
    U = len(rnds)
    rnd = gg20.pack_randomness(rnds)
    ks = gg20.KeySets(engine, keysets)
    try:
        res = gg20.offline_batch(engine, ks, sess, rnd)
        f = {name: gg20.debug_field(engine, name, U) for name in
             ("CK", "CINVP", "FLAGS") + tuple(f"{n}{x}" for n in ("S", "E", "S1", "GS1", "UV") for x in range(3))}
    finally:
        ks.free()
    inverted = f["FLAGS"].view(np.uint8)[:, 3]
    assert 0 < inverted.sum() < U                              # both outcomes of the round-1 inversion occur
    for u in range(U):
        pu = u ^ 1
        N = peer_keys[u].p * peer_keys[u].q
        NN = N * N
        cinv = _int(f["CINVP"][u])
        if inverted[u]:
            assert cinv * _int(f["CK"][pu]) % NN == 1, u
        for x in range(3):
            s, e, s1 = _int(f[f"S{x}"][pu]), _int(f[f"E{x}"][pu]), _int(f[f"S1{x}"][pu])
            assert _int(f[f"GS1{x}"][u]) == s1 * N + 1
            want = pow(s, N, NN) * pow(cinv, e, NN) * (s1 * N + 1) % NN
            assert _int(f[f"UV{x}"][u]) == want, (u, x, s % peer_keys[u].p == 0, s % peer_keys[u].q == 0)
    _assert_matches_twin(res, _twin(keysets, sess, rnd), range(len(sess)))


def test_peer_u_prime_moves_work_off_the_nadic_list(engine):
    from mpecdsa_b200 import gg20
    keysets = fixtures.load_all_keysets()
    sess, rnd = gg20.synthetic_batch(keysets, 256, 0x5E55)
    ks = gg20.KeySets(engine, keysets)
    try:
        engine.work(reset=True)
        res = gg20.offline_batch(engine, ks, sess, rnd)
        per_unit = engine.work() / (2 * len(sess))
        prof = engine.profile_step(lambda: gg20.offline_batch(engine, ks, sess, rnd))
    finally:
        ks.free()
    assert not res.status.any()
    assert per_unit <= PARENT_MAC32_PER_UNIT - 60e6, per_unit
    launches = lambda prefix: sum(v["launches"] for k, v in prof.items() if k.startswith(prefix))
    assert launches("nadic_jobs_kernel<64") == 5, prof
    assert launches("nadic_jobs_kernel<32") == PARENT_PADIC_LAUNCHES + 1, prof
