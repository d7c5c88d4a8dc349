"""TEST INFRASTRUCTURE: GG20 `Keygen` Round0..Round4 (/root/reference/src/protocols/multi_party_ecdsa/gg_2020/state_machine/keygen/
rounds.rs:26-300) for one group, restated party by party from the per-phase functions of oracle/keygen_oracle.py.  Every receiver
runs every verification itself (the reference's `into_vec_including_me`), so the once-per-sender shortcut of
`tecdsa_gg20_keygen_batch` is checked here: the receivers must agree.  Also the CPU helpers the keygen tests share: deterministic
prime pairs and seeded inputs."""
from __future__ import annotations

import random
from dataclasses import dataclass
from math import gcd
from typing import Dict, List, Optional, Sequence, Tuple

from oracle import gg20_oracle as o
from oracle import keygen_oracle as kg

Q = o.Q
ST_OK, ST_INVALID_KEY, ST_NOT_INVERTIBLE, ST_PROOF, ST_INVALID_SS = 0, 2, 4, 10, 12


@dataclass
class KeygenLocalKey(o.LocalKey):
    """`LocalKey` (keygen/rounds.rs:310-322): the fields of oracle.LocalKey plus the party's own `vss_scheme.commitments`"""
    vss_commitments: List[o.Point] = None


def _correct_key_proof(p: int, q: int) -> List[int]:
    """NiCorrectKeyProof::proof; where N has no inverse mod phi the engine's exponent is 0 (every sigma = 1), which verification rejects"""
    try:
        return kg.correct_key_proof(o.DecryptionKey(p, q))
    except ValueError:
        return [1] * kg.M2


def keygen_group(t: int, n: int, primes: Sequence[Tuple[Tuple[int, int], Tuple[int, int]]], rnd: Sequence[Dict]):
    """primes[i] = ((p, q), (p~, q~)) of party i + 1; rnd[i] = its samples: u, coeffs = [a_1..a_t], blind, h1, xhi, cdl_nonce =
    (r1, r2), dlog_nonce.  -> (keys, status, bad_actors): keys[i] a KeygenLocalKey (None unless the whole group completed),
    status[i] the error party i + 1's `proceed` returns (TECDSA_ST_*), bad_actors[i] its mask (bit j = party j + 1)."""
    status, bad = [ST_OK] * n, [0] * n
    # Round 0 / 1: Keys::create, generate_h1_h2_N_tilde, phase1_broadcast_phase3_proof_of_correct_key_proof_of_correct_h1h2
    for i in range(n):
        pt, qt = primes[i][1]
        if gcd(rnd[i]["xhi"], (pt - 1) * (qt - 1)) != 1:
            status[i] = ST_NOT_INVERTIBLE                     # the reference draws xhi again (party_i.rs:144-149)
    if any(status):
        return [None] * n, status, bad
    bcs, decs = [], []
    for i in range(n):
        (p, q), (pt, qt) = primes[i]
        r = rnd[i]
        nt, h1, h2, xn, xin = kg.h1_h2_n_tilde(pt, qt, r["h1"], r["xhi"])
        st1, st2 = o.DLogStatement(nt, h1, h2), o.DLogStatement(nt, h2, h1)
        y_i = o.pt_mul(o.G, r["u"])
        N = p * q
        bcs.append(kg.KeyGenBroadcast1(o.EncryptionKey(N, N * N), st1, o.hash_commitment(o.bn_from_bytes(o.pt_compress(y_i)), r["blind"]),
                                       _correct_key_proof(p, q), kg.composite_dlog_prove(st1, xn, r["cdl_nonce"][0]),
                                       kg.composite_dlog_prove(st2, xin, r["cdl_nonce"][1])))
        decs.append(kg.KeyGenDecommit1(r["blind"], y_i))
    # Round 2: every receiver checks every broadcast, its own included
    masks = [sum(1 << j for j in range(n) if not kg.phase1_verify(bcs[j], decs[j])) for _ in range(n)]
    assert len(set(masks)) == 1, "receivers disagree on a broadcast"
    if masks[0]:
        return [None] * n, [ST_INVALID_KEY] * n, masks
    vss, shares = zip(*[kg.vss_share(t, n, rnd[j]["u"], rnd[j]["coeffs"]) for j in range(n)])
    y_vec = [d.y_i for d in decs]
    # Round 3: receiver i validates the share every sender j sent it
    shared = []
    for i in range(n):
        mine = [shares[j][i] for j in range(n)]
        bad[i] = sum(1 << j for j in range(n) if not (kg.vss_validate_share(vss[j], mine[j], i + 1) and vss[j].commitments[0] == y_vec[j]))
        if not bad[i]:
            res = kg.phase2_verify_vss(y_vec, mine, list(vss), i + 1, rnd[i]["dlog_nonce"])
            assert res is not None
            shared.append(res)
    if any(bad):
        return [None] * n, [ST_INVALID_SS if m else ST_OK for m in bad], bad
    proofs = [s[2] for s in shared]
    # Round 4: every receiver checks every DLog proof against the commitments to x_j
    xi = kg.commitments_to_xi(list(vss))
    masks = [sum(1 << j for j in range(n) if not (o.dlog_verify(proofs[j]) and xi[j] == proofs[j].pk)) for _ in range(n)]
    assert len(set(masks)) == 1
    if masks[0]:
        return [None] * n, [ST_PROOF] * n, masks
    assert all(kg.verify_dlog_proofs_check_against_vss(proofs, list(vss)) for _ in range(n))
    y_sum = y_vec[0]
    for y in y_vec[1:]:
        y_sum = o.pt_add(y_sum, y)
    keys = [KeygenLocalKey(i=i + 1, t=t, n=n, x_i=shared[i][1], dk=o.DecryptionKey(*primes[i][0]), pk_vec=[pf.pk for pf in proofs],
                           paillier_key_vec=[b.e for b in bcs], h1_h2_n_tilde_vec=[b.dlog_statement for b in bcs], y_sum_s=y_sum,
                           vss_commitments=list(vss[i].commitments)) for i in range(n)]
    return keys, status, bad


# ------------------------------------------------------------------------------------------------ shared test inputs
_SMALL = [p for p in range(3, 2000) if all(p % d for d in range(2, int(p ** 0.5) + 1))]


def _is_probable_prime(c: int, rng: random.Random) -> bool:
    if any(c % s == 0 for s in _SMALL):
        return c in _SMALL
    d, r = c - 1, 0
    while d % 2 == 0:
        d, r = d // 2, r + 1
    for _ in range(24):
        x = pow(rng.randrange(2, c - 1), d, c)
        if x in (1, c - 1):
            continue
        for _ in range(r - 1):
            x = x * x % c
            if x == c - 1:
                break
        else:
            return False
    return True


def prime_pair(seed: int, bits: int = 1024) -> Tuple[int, int]:
    """two distinct primes of `bits` bits whose product has 2 * bits bits, deterministic in the seed"""
    rng = random.Random(seed)
    out = []
    while len(out) < 2:
        c = rng.getrandbits(bits) | (3 << (bits - 2)) | 1
        if c not in out and _is_probable_prime(c, rng):
            out.append(c)
    return out[0], out[1]


def random_inputs(t: int, n_tilde: Tuple[int, int], rng: random.Random) -> Dict:
    """one party's samples, from the reference's ranges, with a Python RNG"""
    pt, qt = n_tilde
    phi = (pt - 1) * (qt - 1)
    while True:
        xhi = rng.randrange(phi)
        if gcd(xhi, phi) == 1:
            break
    return {"u": rng.randrange(1, Q), "coeffs": [rng.randrange(1, Q) for _ in range(t)], "blind": rng.getrandbits(256),
            "h1": rng.randrange(pt * qt), "xhi": xhi, "cdl_nonce": (rng.getrandbits(512), rng.getrandbits(512)), "dlog_nonce": rng.randrange(1, Q)}


def lagrange_at_zero(points: Sequence[Tuple[int, int]]) -> int:
    """the secret from t + 1 (index, share) points"""
    acc = 0
    for i, (xi, yi) in enumerate(points):
        num = den = 1
        for j, (xj, _) in enumerate(points):
            if i != j:
                num, den = num * xj % Q, den * (xj - xi) % Q
        acc = (acc + yi * num * pow(den, -1, Q)) % Q
    return acc
