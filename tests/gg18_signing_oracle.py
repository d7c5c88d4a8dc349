"""CPU restatement of GG18 signing for any signing set (gg_2018/test.rs `sign`, /root/reference/src/protocols/multi_party_ecdsa/
gg_2018/test.rs:163-403), the comparator of tecdsa_gg18_signing_batch, and of the seeded draw of its inputs (gg18.sample_inputs).
It composes the phase functions of oracle/gg18_oracle.py with the MtA of oracle/gg20_oracle.py under an empty statement list, party
by party: every receiver runs every check itself (no check is shared between receivers).  A session stops at the end of the first
phase in which any signer failed; phases are those of the call's status table (MessageB, get_alpha, 3, 4, 5a, 5c, 5d, output).

TEST INFRASTRUCTURE ONLY: imported by tests/ and tools/ and nothing else.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

from oracle import gg18_oracle as g18
from oracle import seeded_sampling as ss
from oracle.gg20_oracle import G, Q, Point, lagrange_at_zero, message_a, message_b, pt_mul, verify_proofs_get_alpha

OK, INVALID_KEY, NOT_INVERTIBLE, INVALID_SIG, COMMITMENT = 0, 2, 4, 9, 11

ELEMENT_FIELDS = ("k", "gamma", "blind", "r_a", "l", "rho", "blind5", "blind5c", "heg_s1", "heg_s2", "dlog_nonce")
PAIR_FIELDS = ("beta_tag_gamma", "r_gamma", "beta_tag_w", "r_w", "nonce_gamma_b", "nonce_gamma_beta", "nonce_w_b", "nonce_w_beta")
STREAMS = {f: 80 + i for i, f in enumerate(ELEMENT_FIELDS + PAIR_FIELDS)}          # TECDSA_RNDS_G18_*


@dataclass
class SignerRandomness:
    """Every value one signer samples; the per-peer lists are ordered by j = 0..ttag-2 (peer position `ind(j)`)."""
    k: int = 0
    gamma: int = 0
    blind: int = 0
    r_a: int = 0
    l: int = 0
    rho: int = 0
    blind5: int = 0
    blind5c: int = 0
    heg_s1: int = 0
    heg_s2: int = 0
    dlog_nonce: int = 0
    beta_tag_gamma: List[int] = field(default_factory=list)
    r_gamma: List[int] = field(default_factory=list)
    beta_tag_w: List[int] = field(default_factory=list)
    r_w: List[int] = field(default_factory=list)
    nonce_gamma_b: List[int] = field(default_factory=list)
    nonce_gamma_beta: List[int] = field(default_factory=list)
    nonce_w_b: List[int] = field(default_factory=list)
    nonce_w_beta: List[int] = field(default_factory=list)


@dataclass
class SessionResult:
    status: List[int]
    R: List[Optional[Point]]                              # per signer; None unless the session completed
    signature: Optional[Tuple[int, int, int]] = None      # (r, s, recid)
    phase: int = -1                                       # the phase in which the session stopped (-1: complete)
    sigma: List[int] = field(default_factory=list)        # sigma_i per signer (phase 2 onwards), for the algebraic checks
    delta: List[int] = field(default_factory=list)


def _ind(i: int, j: int) -> int:
    return j if j < i else j + 1


def sign_session(keys: Sequence, s_l: Sequence[int], rnd: Sequence[SignerRandomness], message: int) -> SessionResult:
    """All signers of one session in lock step.  keys[p] / rnd[p] belong to signer position p (keys: LocalKeys of oracle/gg20_oracle.py;
    only dk, paillier_key_vec, x_i and y_sum_s are read); s_l[p] is its 1-based keygen index; message the hashed message."""
    T = len(s_l)
    l_s = [x - 1 for x in s_l]
    status = [OK] * T
    res = SessionResult(status, [None] * T)

    def stop(phase):
        if any(status):
            res.phase = phase
            return True
        return False

    w = [lagrange_at_zero(l_s[p], l_s) * keys[p].x_i % Q for p in range(T)]                  # SignKeys::create
    k = [r.k % Q for r in rnd]
    gamma = [r.gamma % Q for r in rnd]
    y = keys[0].y_sum_s
    # ---- phase 1: commitment to g^gamma_i, MessageA = Enc(k_i) without range proofs
    g_gamma = [pt_mul(G, x) for x in gamma]
    com = [g18.phase1_broadcast(g_gamma[p], rnd[p].blind) for p in range(T)]
    m_a = [message_a(k[p], keys[p].paillier_key_vec[l_s[p]], rnd[p].r_a, [], []) for p in range(T)]
    # ---- phase 2: MessageB for gamma_i and w_i towards every peer under the peer's key (sender p, receiver ind(p, j))
    m_b_g = [[None] * (T - 1) for _ in range(T)]
    m_b_w = [[None] * (T - 1) for _ in range(T)]
    beta = [[0] * (T - 1) for _ in range(T)]
    nu = [[0] * (T - 1) for _ in range(T)]
    for p in range(T):
        r = rnd[p]
        for j in range(T - 1):
            a = _ind(p, j)
            ek = keys[p].paillier_key_vec[l_s[a]]
            rb = message_b(gamma[p], ek, m_a[a], r.r_gamma[j], r.beta_tag_gamma[j], [], r.nonce_gamma_b[j], r.nonce_gamma_beta[j])
            rw = message_b(w[p], ek, m_a[a], r.r_w[j], r.beta_tag_w[j], [], r.nonce_w_b[j], r.nonce_w_beta[j])
            if rb is None or rw is None:
                status[p] = INVALID_KEY
                break
            m_b_g[p][j], beta[p][j] = rb
            m_b_w[p][j], nu[p][j] = rw
    if stop(0):
        return res
    recv = lambda table, p, b: table[b][p if p < b else p - 1]          # what receiver p got from sender b
    delta, sigma = [0] * T, [0] * T
    for p in range(T):
        alphas, mus = [], []
        for j in range(T - 1):
            b = _ind(p, j)
            ra = verify_proofs_get_alpha(recv(m_b_g, p, b), keys[p].dk, k[p])
            rm = verify_proofs_get_alpha(recv(m_b_w, p, b), keys[p].dk, k[p])
            if ra is None or rm is None:
                status[p] = INVALID_KEY
                break
            alphas.append(ra[0]); mus.append(rm[0])
        else:
            delta[p] = g18.phase2_sum(k[p], gamma[p], alphas, beta[p])
            sigma[p] = g18.phase2_sum(k[p], w[p], mus, nu[p])
    res.delta, res.sigma = delta, sigma
    if stop(1):
        return res
    # ---- phase 3
    dinv = g18.phase3_reconstruct_delta(delta)
    if dinv is None:
        status[:] = [NOT_INVERTIBLE] * T
    if stop(2):
        return res
    # ---- phase 4: each signer checks every decommitment and the key of every MessageB(gamma) it received
    R = [None] * T
    for p in range(T):
        pks = [g_gamma[p] if x == p else recv(m_b_g, p, x).b_proof.pk for x in range(T)]
        R[p] = g18.phase4(dinv, pks, [(rnd[x].blind, g_gamma[x]) for x in range(T)], com)
        if R[p] is None:
            status[p] = INVALID_KEY
    if stop(3):
        return res
    # ---- phase 5
    s_i = [g18.phase5_local_sig(k[p], message, R[p], sigma[p]) for p in range(T)]
    a5 = [None] * T
    for p in range(T):
        r = rnd[p]
        if any(v % Q == 0 for v in (r.l, r.rho, r.heg_s2, r.dlog_nonce)):          # Scalar::random() != 0: no identity points
            status[p] = INVALID_KEY
            continue
        a5[p] = g18.phase5a(s_i[p], r.l % Q, r.rho % Q, R[p], r.blind5, r.heg_s1 % Q, r.heg_s2 % Q, r.dlog_nonce % Q)
        if a5[p].V is None or a5[p].heg.T is None:
            status[p] = INVALID_KEY
    if stop(4):
        return res
    c5 = [None] * T
    for p in range(T):
        r = rnd[p]
        code, c5[p] = g18.phase5c(message, R[p], y, r.rho % Q, r.l % Q, [a5[x] for x in range(T) if x != p], a5[p].V, r.blind5c)
        status[p] = code
    if stop(5):
        return res
    decom2 = [(c5[p][1], c5[p][2], rnd[p].blind5c) for p in range(T)]
    com2 = [c5[p][0] for p in range(T)]
    for p in range(T):
        status[p] = g18.phase5d(decom2, com2, [a.B for a in a5])
    if stop(6):
        return res
    sig = [None] * T
    for p in range(T):
        status[p], sig[p] = g18.output_signature(R[p], y, message, s_i)
    if stop(7):
        return res
    res.R, res.signature = R, sig[0]
    return res


def sign_sessions(keysets: Sequence[Sequence], sessions: Sequence[Sequence[int]], rnd: Sequence[SignerRandomness], messages: Sequence[int]) -> List[SessionResult]:
    """sign_session over descriptors [n][1 + T] (key set, then s_l[p] - 1) as tecdsa_gg18_signing_batch takes them; rnd per element
    u = s * T + p."""
    out = []
    for s, d in enumerate(sessions):
        T = len(d) - 1
        out.append(sign_session([keysets[d[0]][i] for i in d[1:]], [i + 1 for i in d[1:]], rnd[s * T:(s + 1) * T], messages[s]))
    return out


def sample_inputs(seed: bytes, n_rows: Sequence[int], parties: int, signers: int, sessions: Sequence[Sequence[int]], elements=None) -> Dict[int, SignerRandomness]:
    """gg18.sample_inputs restated over oracle/seeded_sampling.py: stream TECDSA_RNDS_G18_<field>, element id (sub << 32) | u (sub = 0
    per element, the peer index j per pair), kinds of tecdsa_gg18_signing_in.  n_rows = the Paillier N of every key row of the key
    sets.  -> {u: SignerRandomness} for the elements listed (all by default)."""
    T = signers
    E = len(sessions) * T
    own = [sessions[u // T][0] * parties + sessions[u // T][1 + u % T] for u in range(E)]

    def draw(f, u, sub=0, kind="scalar", bound=0, bits=0):
        v, ok, _ = ss.sample(seed, STREAMS[f], (sub << 32) | u, kind, bound=bound, bits=bits)
        assert ok, (f, u, sub)
        return v

    out = {}
    for u in (range(E) if elements is None else elements):
        r = SignerRandomness()
        for f in ("k", "gamma", "l", "rho", "heg_s1", "heg_s2", "dlog_nonce"):
            setattr(r, f, draw(f, u))
        for f in ("blind", "blind5", "blind5c"):
            setattr(r, f, draw(f, u, kind="bits", bits=256))
        r.r_a = draw("r_a", u, kind="below", bound=n_rows[own[u]])
        for j in range(T - 1):
            peer = own[u - u % T + _ind(u % T, j)]
            for f in ("beta_tag_gamma", "r_gamma", "beta_tag_w", "r_w"):
                getattr(r, f).append(draw(f, u, j, "below", n_rows[peer]))
            for f in ("nonce_gamma_b", "nonce_gamma_beta", "nonce_w_b", "nonce_w_beta"):
                getattr(r, f).append(draw(f, u, j))
        out[u] = r
    return out
