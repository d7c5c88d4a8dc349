"""GG20 offline stage for ANY signing set over the batched L0-L2 calls: the size-generic driver next to the fused L3 call
(`tecdsa_gg20_offline_batch`, which is specialised to the t = 1 / two-signer work unit of SURVEY.md section 8).  Same functions, in the
round order of /root/reference/src/protocols/multi_party_ecdsa/gg_2020/state_machine/sign/rounds.rs:68-636, with the reference's
index convention (`ind = if j < i {j} else {j+1}`); every round is a handful of batch calls over all (session, signer[, peer])
instances.  Element u = session * ttag + position; pair t = u * (ttag - 1) + j is "element u towards its j-th peer".
No arithmetic happens on the host — only index bookkeeping and equality tests.  Oracle: oracle/gg20_general_oracle.py."""
from __future__ import annotations

import ctypes
from typing import Dict, List, Optional, Sequence

import numpy as np

from . import HOST, SAMPLE_BELOW, SAMPLE_BITS, SAMPLE_RANGE1, SAMPLE_SCALAR, SAMPLE_UNIT, Engine, EngineError, _ptr, ints_to_limbs, limbs_to_ints
from . import gg18, gg20
from .gg20 import KeySets, unpack_point

ST_INVALID_KEY, ST_PDL, ST_PHASE5, ST_PHASE6, ST_PROOF, ST_COMMIT = 2, 6, 7, 8, 10, 11


def _pts_of(a: np.ndarray):
    return [unpack_point(v) for v in limbs_to_ints(a)]


def sample_rnd(eng: Engine, keys: KeySets, ttag: int, key_rows: Sequence[int], all_rows: Sequence[Sequence[int]], seed: Optional[bytes] = None) -> Dict[str, list]:
    """The `rnd` dictionary `offline_batch` takes, every value drawn on the device as the reference draws it inside `MessageA::a`,
    `MessageB::b`, `AliceProof::generate`, `PDLwSlackProof::prove` and `SignKeys::create` (ranges: oracle/sampling.py::sample_unit),
    one `Engine.sample` call per field.  Streams are the TECDSA_RNDS_* ids of the fused call's record (`gg20.RNDS`; the Alice fields
    use RNDS_ALICE + part for every statement).  Element id = (sub << 32) | u for element u = session * ttag + position, with sub =
    0 for the per-element fields, the statement index x for alice[u][x], and the peer index j for the per-pair fields of pair
    u * (ttag - 1) + j — so no (stream, id) repeats inside a call.  seed=None draws a fresh seed; a seed serves ONE call."""
    seed = gg20.fresh_seed(seed)
    U, P1 = len(key_rows), ttag - 1
    q = gg20._Q
    N, NT = keys.table(0, 64), keys.table(2, 64)
    peer_row = [[key_rows[u // ttag * ttag + (j if j < u % ttag else j + 1)] for u in range(U)] for j in range(P1)]

    def draw(kind, name, sub=0, bound=None, bits=0, limbs=None, stream=None):
        vals, st = eng.sample(kind, U, seed, stream=gg20.RNDS[name] if stream is None else stream, first_id=sub << 32, bound=bound, bits=bits, limbs=limbs)
        if st.any():
            raise EngineError(f"sampling {name}: element {int(np.flatnonzero(st)[0])} has status {int(st[st != 0][0])}")
        return vals

    rnd = {f: draw(SAMPLE_SCALAR, f) for f in ("gamma", "k", "l", "ped_s1", "ped_s2", "heg_s1", "heg_s2")}
    rnd["blind"] = draw(SAMPLE_BITS, "blind", bits=256)
    n_own = [N[r] for r in key_rows]
    rnd["r_k"] = draw(SAMPLE_BELOW, "r_k", bound=n_own)
    n_st = len(all_rows[0]) if U else 0
    per_st = []
    for x in range(n_st):
        nt = [NT[all_rows[u][x]] for u in range(U)]
        A = gg20.RNDS_ALICE
        per_st.append((draw(SAMPLE_BELOW, "alice alpha", x, [q ** 3] * U, stream=A), draw(SAMPLE_UNIT, "alice beta", x, n_own, stream=A + 1),
                       draw(SAMPLE_BELOW, "alice gamma", x, [q ** 3 * v for v in nt], stream=A + 2), draw(SAMPLE_BELOW, "alice rho", x, [q * v for v in nt], stream=A + 3)))
    rnd["alice"] = [[tuple(part[u] for part in per_st[x]) for x in range(n_st)] for u in range(U)]
    per_pair = {f: [None] * (U * P1) for f in ("beta_tag_gamma", "r_gamma", "nonce_gamma_b", "nonce_gamma_beta", "beta_tag_w", "r_w", "nonce_w_b", "nonce_w_beta", "pdl")}
    for j in range(P1):
        n_peer, nt_peer = [N[r] for r in peer_row[j]], [NT[r] for r in peer_row[j]]
        cols = {f: draw(SAMPLE_BELOW, f, j, n_peer) for f in ("beta_tag_gamma", "r_gamma", "beta_tag_w", "r_w")}
        cols.update({f: draw(SAMPLE_SCALAR, f, j) for f in ("nonce_gamma_b", "nonce_gamma_beta", "nonce_w_b", "nonce_w_beta")})
        pdl = (draw(SAMPLE_BELOW, "pdl_alpha", j, [q ** 3] * U), draw(SAMPLE_RANGE1, "pdl_beta", j, n_own), draw(SAMPLE_BELOW, "pdl_rho", j, [q * v for v in nt_peer]),
               draw(SAMPLE_BELOW, "pdl_gamma", j, [q ** 3 * v for v in nt_peer]))
        for u in range(U):
            for f, col in cols.items():
                per_pair[f][u * P1 + j] = col[u]
            per_pair["pdl"][u * P1 + j] = tuple(p[u] for p in pdl)
    rnd.update(per_pair)
    return rnd


def offline_batch(eng: Engine, keys: KeySets, ttag: int, key_rows: Sequence[int], all_rows: Sequence[Sequence[int]], w: Sequence[int],
                  g_w: Sequence, y: Sequence, rnd: Dict[str, list], messages: bool = False) -> Dict[str, list]:
    """`OfflineStage` Round0..Round6 for sessions of `ttag` signers.
    key_rows[u]  key row (Paillier key + N~/h1/h2 setup) of element u in `keys`;
    all_rows[u]  the key rows of ALL keygen parties of its key, in keygen order (the statements `MessageA::a` proves against);
    w[u], g_w[u] the Lagrange-weighted share and its public image (`SignKeys::g_w_vec`), y[u] the public key;
    rnd          per element: gamma, k, blind, r_k, l, ped_s1, ped_s2, heg_s1, heg_s2 and alice[u] = n tuples (alpha, beta, gamma, ro);
                 per pair: beta_tag_gamma, r_gamma, nonce_gamma_b, nonce_gamma_beta, beta_tag_w, r_w, nonce_w_b, nonce_w_beta and
                 pdl[t] = (alpha, beta, rho, gamma).
    -> dict(status, R, sigma, k, T): `CompletedOfflineStage` per element (T = its own T_i); status = the reference's first error.
    With messages=True also "messages": per element the list of `Msg<OfflineProtocolMessage>` documents it sends (serde-JSON shape of
    state_machine/sign.rs:478-490 through wire.py; sender / receiver = 1-based signer positions), for sessions that completed."""
    U, P1 = len(key_rows), ttag - 1
    status = np.zeros(U, np.uint8)
    sess = lambda u: u // ttag * ttag
    peer = [sess(u) + (j if j < u % ttag else j + 1) for u in range(U) for j in range(P1)]       # pair t -> the other element
    me = [u for u in range(U) for _ in range(P1)]
    back = {(me[t], peer[t]): t for t in range(U * P1)}                                          # (from, to) -> pair index

    stopped = set()                      # sessions in which some party failed in an EARLIER round: nothing more is recorded for them

    def fail(elems, code):
        for u in elems:
            if not status[u] and sess(u) not in stopped:
                status[u] = code

    def end_round():
        stopped.update(sess(u) for u in range(U) if status[u])

    def session_ok(u):
        return not status[sess(u):sess(u) + ttag].any()

    k, gamma = list(rnd["k"]), list(rnd["gamma"])
    # ---- Round 0: commitment to g^gamma, MessageA with one range proof per keygen party
    g_gamma = eng.secp_mul(None, gamma)
    com = gg20.hash_commitment(eng, g_gamma, rnd["blind"])
    c_a, proofs = gg20.mta_message_a(eng, keys, list(key_rows), [list(r) for r in all_rows], k, rnd["r_k"], rnd["alice"])
    # ---- Round 1: element `me` answers peer's MessageA twice (b = gamma, b = w) under the PEER's Paillier key
    a_rows = [key_rows[v] for v in peer]
    a_st = [list(all_rows[u]) for u in me]
    a_ca = [c_a[v] for v in peer]
    a_pf = {f: [proofs[f][v] for v in peer] for f in proofs}
    cb_g, bp_g, btp_g, beta_g, st = gg20.mta_message_b(eng, keys, a_rows, a_st, [gamma[u] for u in me], a_ca, a_pf, rnd["r_gamma"], rnd["beta_tag_gamma"],
                                                        rnd["nonce_gamma_b"], rnd["nonce_gamma_beta"])
    fail([me[t] for t in range(U * P1) if st[t]], ST_INVALID_KEY)
    cb_w, bp_w, btp_w, beta_w, st = gg20.mta_message_b(eng, keys, a_rows, a_st, [w[u] for u in me], a_ca, a_pf, rnd["r_w"], rnd["beta_tag_w"],
                                                        rnd["nonce_w_b"], rnd["nonce_w_beta"])
    fail([me[t] for t in range(U * P1) if st[t]], ST_INVALID_KEY)
    end_round()
    # ---- Round 2: alice = peer[t] opens what bob = me[t] sent her
    al_rows = [key_rows[v] for v in peer]
    al_k = [k[v] for v in peer]
    alpha_g, _, st = gg20.mta_get_alpha(eng, keys, al_rows, al_k, cb_g, bp_g, btp_g)
    fail([peer[t] for t in range(U * P1) if st[t]], ST_INVALID_KEY)
    alpha_w, _, st = gg20.mta_get_alpha(eng, keys, al_rows, al_k, cb_w, bp_w, btp_w)
    fail([peer[t] for t in range(U * P1) if st[t]], ST_INVALID_KEY)
    pk_w = _pts_of(bp_w[:, :16])
    fail([peer[t] for t in range(U * P1) if pk_w[t] != g_w[me[t]]], ST_INVALID_KEY)               # rounds.rs:281
    delta = eng.scalar_op("mul", k, gamma)
    sigma = eng.scalar_op("mul", k, list(w))
    for j in range(P1):
        incoming = [back[(sess(u) + (j if j < u % ttag else j + 1), u)] for u in range(U)]         # the pair in which u is alice of its j-th peer
        delta = eng.scalar_op("add", delta, [alpha_g[t] for t in incoming])
        sigma = eng.scalar_op("add", sigma, [alpha_w[t] for t in incoming])
        delta = eng.scalar_op("add", delta, [beta_g[u * P1 + j] for u in range(U)])
        sigma = eng.scalar_op("add", sigma, [beta_w[u * P1 + j] for u in range(U)])
    T, t_proof = gg20.pedersen_prove(eng, sigma, rnd["l"], rnd["ped_s1"], rnd["ped_s2"])
    end_round()
    # ---- Round 3: every T_i's Pedersen proof, delta^-1
    st = gg20.pedersen_verify(eng, T, t_proof)
    tot = [0] * U
    for j in range(ttag):
        tot = eng.scalar_op("add", tot, [delta[sess(u) + j] for u in range(U)])
    dinv = eng.scalar_op("inv", tot)
    for u in range(U):
        if dinv[u] is None or st[sess(u):sess(u) + ttag].any():
            fail([u], ST_PROOF)
    dinv = [d or 1 for d in dinv]
    end_round()
    # ---- Round 4: decommitments, R, R_dash, one PDL-with-slack proof per peer
    pk_g = _pts_of(bp_g[:, :16])
    pks = [[g_gamma[u] if sess(u) + j == u else pk_g[back[(sess(u) + j, u)]] for j in range(ttag)] for u in range(U)]
    R, st = gg18.phase4(eng, ttag, dinv, pks, g_gamma, rnd["blind"], com)
    fail([u for u in range(U) if st[u]], ST_COMMIT)
    Rs = [p if p is not None else g_gamma[u] for u, p in enumerate(R)]
    R_dash = eng.secp_mul(Rs, k)
    pa, pb, pr, pg = zip(*rnd["pdl"])
    pdl = gg20.pdl_prove(eng, keys, [key_rows[u] for u in me], [key_rows[v] for v in peer], [k[u] for u in me], [rnd["r_k"][u] for u in me],
                         [c_a[u] for u in me], [R_dash[u] for u in me], [Rs[u] for u in me], list(pa), list(pb), list(pr), list(pg))
    end_round()
    # ---- Round 5: every proof of every signer, sum of R_dash, S_i with its consistency proof
    st = gg20.pdl_verify(eng, keys, [key_rows[u] for u in me], [key_rows[v] for v in peer], [c_a[u] for u in me], [R_dash[u] for u in me], [Rs[u] for u in me],
                         pdl["z"], pdl["u1"], pdl["u2"], pdl["u3"], pdl["s1"], pdl["s2"], pdl["s3"])
    bad_sessions = {sess(me[t]) for t in range(U * P1) if st[t]}
    fail([u for u in range(U) if sess(u) in bad_sessions], ST_PDL)
    gen = eng.secp_mul(None, [1])[0]
    acc = [R_dash[sess(u)] for u in range(U)]
    for j in range(1, ttag):
        acc = eng.point_add(acc, [R_dash[sess(u) + j] for u in range(U)])
    fail([u for u in range(U) if acc[u] != gen], ST_PHASE5)
    S = eng.secp_mul(Rs, sigma)
    heg = gg20.heg_prove(eng, Rs, _pts_of(T), S, rnd["l"], sigma, rnd["heg_s1"], rnd["heg_s2"])
    end_round()
    # ---- Round 6
    st = gg20.heg_verify(eng, Rs, _pts_of(T), S, heg)
    acc = [S[sess(u)] for u in range(U)]
    for j in range(1, ttag):
        acc = eng.point_add(acc, [S[sess(u) + j] for u in range(U)])
    for u in range(U):
        if st[sess(u):sess(u) + ttag].any() or acc[u] != y[u]:
            fail([u], ST_PHASE6)
    # a session stops in the round where its first party failed: the other parties of that session produce nothing either
    out_R = [R[u] if session_ok(u) else None for u in range(U)]
    out = {"status": status, "R": out_R, "sigma": sigma, "k": k, "T": _pts_of(T), "session_ok": [session_ok(u) for u in range(U)]}
    if messages:
        from . import wire
        E = wire.DEFAULT
        Tp = _pts_of(T)
        docs = []
        for u in range(U):
            if not session_ok(u):
                docs.append([])
                continue
            me_pos = u % ttag + 1
            n_st = len(all_rows[u])
            rp = [{f: proofs[f][u][x] for f in ("z", "e", "s", "s1", "s2")} for x in range(n_st)]
            ped = wire.pedersen_proof(t_proof[u]); ped["com"] = E.point(Tp[u])
            m = [wire.msg(me_pos, None, wire.offline_message("M1", [wire.message_a(c_a[u], rp), wire.sign_broadcast_phase1(com[u])]))]
            for j in range(P1):
                t = u * P1 + j
                m.append(wire.msg(me_pos, peer[t] % ttag + 1, wire.offline_message("M2", [wire.message_b(cb_g[t], bp_g[t], btp_g[t]), wire.message_b(cb_w[t], bp_w[t], btp_w[t])])))
            m.append(wire.msg(me_pos, None, wire.offline_message("M3", [E.scalar(delta[u]), E.point(Tp[u]), ped])))
            m.append(wire.msg(me_pos, None, wire.offline_message("M4", wire.sign_decommit_phase1(rnd["blind"][u], g_gamma[u]))))
            pl = [wire.pdl_proof({f: pdl[f][u * P1 + j] for f in ("z", "u1", "u2", "u3", "s1", "s2", "s3")}) for j in range(P1)]
            m.append(wire.msg(me_pos, None, wire.offline_message("M5", [E.point(R_dash[u]), pl])))
            m.append(wire.msg(me_pos, None, wire.offline_message("M6", [E.point(S[u]), wire.heg_proof(heg[u])])))
            docs.append(m)
        out["messages"] = docs
    return out


# ----------------------------------------------------------------------------- the one-call path (tecdsa_gg20_offline_general_batch)
# widths (limbs) of the inputs: per element, per statement of MessageA's range proofs ([parties][E][w]), per pair ([signers-1][E][w])
ELEMENT_FIELDS = {"gamma": 8, "k": 8, "blind": 8, "r_k": 64, "l": 8, "ped_s1": 8, "ped_s2": 8, "heg_s1": 8, "heg_s2": 8}
STATEMENT_FIELDS = {"alice_alpha": 24, "alice_beta": 64, "alice_gamma": 88, "alice_rho": 72}
PAIR_FIELDS = {"beta_tag_gamma": 64, "r_gamma": 64, "nonce_gamma_b": 8, "nonce_gamma_beta": 8, "beta_tag_w": 64, "r_w": 64, "nonce_w_b": 8,
               "nonce_w_beta": 8, "pdl_alpha": 24, "pdl_beta": 64, "pdl_rho": 72, "pdl_gamma": 88}
IN_FIELDS = list(ELEMENT_FIELDS) + list(STATEMENT_FIELDS) + list(PAIR_FIELDS)


class _GeneralIn(ctypes.Structure):
    _fields_ = [(n, ctypes.c_void_p) for n in IN_FIELDS]


class _GeneralOut(ctypes.Structure):
    _fields_ = [(n, ctypes.c_void_p) for n in ("status", "R", "sigma", "T", "complete")]


def _descriptors(sessions, signers: int) -> np.ndarray:
    """[n][1 + signers] uint32 on the host (a CUDA tensor is copied back: the descriptors are public)"""
    from .keygen import _host
    return np.ascontiguousarray(_host(sessions) if not isinstance(sessions, (list, tuple)) else np.asarray(sessions), dtype=np.uint32).reshape(-1, 1 + signers)


def sample_inputs(eng: Engine, keys: KeySets, signers: int, sessions, seed: Optional[bytes] = None, mem: int = HOST) -> Dict[str, object]:
    """Every input of `offline_device`, drawn by `tecdsa_sample_batch` on the stream and element ids `sample_rnd` uses, so the values
    are the ones `sample_rnd` draws from the same seed: element u = session * signers + position has element id (sub << 32) | u,
    sub = the statement x for the range-proof fields and the peer index j for the per-pair fields.  sessions = [n][1 + signers]
    (key set, then s_l[p] - 1).  -> dict field -> array in the layout of tecdsa_offline_general_in (numpy for HOST; CUDA tensors for
    DEVICE, which never reach the host).  seed=None draws a fresh seed; a seed serves ONE call."""
    from .keygen import _buffer, _host, _upload
    from . import seed_words
    lib = eng.lib
    if not getattr(lib, "_sample_bound", False):
        V, S_, I_ = ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int
        lib.tecdsa_sample_batch.argtypes = [V, V, ctypes.c_uint64, ctypes.c_uint32, I_, I_, V, V, S_, I_, V, V, S_, I_]
        lib._sample_bound = True
    d = _descriptors(sessions, signers)
    T, P, n = signers, keys.parties, d.shape[0]
    E, q = n * T, gg20._Q
    # bound tables per key row (public key material) and the key row each element draws under
    N, NT = keys.table(0, 64), keys.table(2, 64)
    tabs = {"N": _upload(ints_to_limbs(N, 64), mem, eng.device), "QNT": _upload(ints_to_limbs([q * v for v in NT], 72), mem, eng.device),
            "Q3NT": _upload(ints_to_limbs([q ** 3 * v for v in NT], 88), mem, eng.device), "Q3": _upload(ints_to_limbs([q ** 3], 24), mem, eng.device)}
    own = (d[:, :1] * P + d[:, 1:]).reshape(E).astype(np.uint32)
    pos = np.arange(E) % T
    base = np.arange(E) - pos

    def peer_rows(j):
        return own[base + np.where(j < pos, j, j + 1)].astype(np.uint32)

    sw = seed_words(gg20.fresh_seed(seed))

    def draw(out, name, kind, stream, sub=0, tab=None, idx=None, bits=0):
        limbs = out.shape[-1]
        st = _buffer((E,), np.uint8, mem, eng.device)
        ix = None if idx is None else _upload(np.asarray(idx, dtype=np.uint32), mem, eng.device)
        nb = 0 if tab is None else tab.shape[0]
        eng._ck(lib.tecdsa_sample_batch(eng._ctx, _ptr(sw), sub << 32, stream, kind, bits, _ptr(tab), _ptr(ix), nb, limbs, _ptr(out), _ptr(st), E, mem),
                "sample_batch")
        bad = np.flatnonzero(_host(st))
        if bad.size:
            raise EngineError(f"sampling {name}: element {int(bad[0])} has status {int(_host(st)[bad[0]])}")

    inp = {f: _buffer((E, w), np.uint32, mem, eng.device) for f, w in ELEMENT_FIELDS.items()}
    inp.update({f: _buffer((P, E, w), np.uint32, mem, eng.device) for f, w in STATEMENT_FIELDS.items()})
    inp.update({f: _buffer((T - 1, E, w), np.uint32, mem, eng.device) for f, w in PAIR_FIELDS.items()})
    zero = np.zeros(E, np.uint32)
    A = gg20.RNDS_ALICE
    try:
        for f in ("gamma", "k", "l", "ped_s1", "ped_s2", "heg_s1", "heg_s2"):
            draw(inp[f], f, SAMPLE_SCALAR, gg20.RNDS[f])
        draw(inp["blind"], "blind", SAMPLE_BITS, gg20.RNDS["blind"], bits=256)
        draw(inp["r_k"], "r_k", SAMPLE_BELOW, gg20.RNDS["r_k"], tab=tabs["N"], idx=own)
        for x in range(P):
            st_rows = (d[:, :1] * P + x).repeat(T, axis=1).reshape(E).astype(np.uint32)
            draw(inp["alice_alpha"][x], "alice alpha", SAMPLE_BELOW, A, x, tabs["Q3"], zero)
            draw(inp["alice_beta"][x], "alice beta", SAMPLE_UNIT, A + 1, x, tabs["N"], own)
            draw(inp["alice_gamma"][x], "alice gamma", SAMPLE_BELOW, A + 2, x, tabs["Q3NT"], st_rows)
            draw(inp["alice_rho"][x], "alice rho", SAMPLE_BELOW, A + 3, x, tabs["QNT"], st_rows)
        for j in range(T - 1):
            pr = peer_rows(j)
            for f in ("beta_tag_gamma", "r_gamma", "beta_tag_w", "r_w"):
                draw(inp[f][j], f, SAMPLE_BELOW, gg20.RNDS[f], j, tabs["N"], pr)
            for f in ("nonce_gamma_b", "nonce_gamma_beta", "nonce_w_b", "nonce_w_beta"):
                draw(inp[f][j], f, SAMPLE_SCALAR, gg20.RNDS[f], j)
            draw(inp["pdl_alpha"][j], "pdl_alpha", SAMPLE_BELOW, gg20.RNDS["pdl_alpha"], j, tabs["Q3"], zero)
            draw(inp["pdl_beta"][j], "pdl_beta", SAMPLE_RANGE1, gg20.RNDS["pdl_beta"], j, tabs["N"], own)
            draw(inp["pdl_rho"][j], "pdl_rho", SAMPLE_BELOW, gg20.RNDS["pdl_rho"], j, tabs["QNT"], pr)
            draw(inp["pdl_gamma"][j], "pdl_gamma", SAMPLE_BELOW, gg20.RNDS["pdl_gamma"], j, tabs["Q3NT"], pr)
    finally:
        sw[:] = 0
    return inp


def offline_device(eng: Engine, keys: KeySets, signers: int, sessions, inp: Dict[str, object], mem: int = HOST, out: Optional[Dict[str, object]] = None,
                   check: bool = True) -> Dict[str, object]:
    """`OfflineStage` Round0..Round6 for every session as ONE call (tecdsa_gg20_offline_general_batch).  sessions = [n][1 + signers];
    inp = the dict `sample_inputs` returns (or the same fields from elsewhere).  -> dict(status [E], R [E][16], sigma [E][8],
    T [E][16], complete [n]): numpy arrays for HOST, CUDA tensors for DEVICE (the caller's, when `out` holds them; sessions is then a
    CUDA tensor too).  A session that did not complete has zero R, sigma and T.  check=False returns the call's rc instead of raising."""
    from .keygen import _buffer
    lib = eng.lib
    if not getattr(lib, "_general_bound", False):
        V = ctypes.c_void_p
        lib.tecdsa_gg20_offline_general_batch.argtypes = [V, V, ctypes.c_int, ctypes.c_size_t, ctypes.c_int, V, ctypes.POINTER(_GeneralIn), ctypes.POINTER(_GeneralOut)]
        lib._general_bound = True
    if mem == HOST:
        sessions = _descriptors(sessions, signers)
        inp = {f: np.ascontiguousarray(v, dtype=np.uint32) for f, v in inp.items()}
    n = sessions.shape[0]
    E = n * signers
    if out is None:
        out = {"status": _buffer((E,), np.uint8, mem, eng.device), "R": _buffer((E, 16), np.uint32, mem, eng.device),
               "sigma": _buffer((E, 8), np.uint32, mem, eng.device), "T": _buffer((E, 16), np.uint32, mem, eng.device),
               "complete": _buffer((n,), np.uint8, mem, eng.device)}
    gi = _GeneralIn(*[_ptr(inp[f]) for f in IN_FIELDS])
    go = _GeneralOut(*[_ptr(out[f]) for f in ("status", "R", "sigma", "T", "complete")])
    rc = lib.tecdsa_gg20_offline_general_batch(eng._ctx, keys.handle, signers, n, mem, _ptr(sessions), ctypes.byref(gi), ctypes.byref(go))
    if not check:
        return rc
    eng._ck(rc, "gg20_offline_general_batch")
    return out


def sign_batch(eng: Engine, signers: int, message, R, sigma, k, y) -> Dict[str, np.ndarray]:
    """GG20's online step (`phase7_local_sig` + `output_signature` + `verify`, party_i.rs:850-936) for completed sessions of
    `signers` signers, on the existing GG18 entry points: s_i = m k_i + r sigma_i is `tecdsa_gg18_local_sig_batch`, and the sum with
    low-s normalisation, recid and verification against y is `tecdsa_gg18_output_signature_batch` — the same arithmetic as GG18's
    party_i.rs:486-730, so no entry point of its own is needed.  message [n] ints (reduced mod q), R [E][16], sigma [E][8], k [E][8]
    (limb rows), y [n] points (y_sum_s).  -> dict(s_i [E][8], r [E][8], s [E][8], recid [E], status [E]) per element: every signer
    derives the session's signature."""
    from . import gg18
    gg18._bind(eng.lib)
    lib = eng.lib
    R, sigma, k = (np.ascontiguousarray(a, dtype=np.uint32) for a in (R, sigma, k))
    E = R.shape[0]
    n = E // signers
    msg = ints_to_limbs([int(message[u // signers]) for u in range(E)], 8)
    Y = ints_to_limbs([gg20.pack_point(y[u // signers]) for u in range(E)], 16)
    s_i, r, s = np.zeros((E, 8), np.uint32), np.zeros((E, 8), np.uint32), np.zeros((E, 8), np.uint32)
    recid, status = np.zeros(E, np.uint8), np.full(E, 255, np.uint8)
    eng._ck(lib.tecdsa_gg18_local_sig_batch(eng._ctx, _ptr(msg), _ptr(R), _ptr(k), _ptr(sigma), _ptr(s_i), E, HOST), "gg18_local_sig")
    eng._ck(lib.tecdsa_gg18_output_signature_batch(eng._ctx, signers, _ptr(R), _ptr(Y), _ptr(msg), _ptr(s_i), _ptr(r), _ptr(s), _ptr(recid), _ptr(status), n, HOST),
            "gg18_output_signature")
    return {"s_i": s_i, "r": r, "s": s, "recid": recid, "status": status}
