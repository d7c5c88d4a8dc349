"""Host-side mirror of the GG18 signing phases that GG20 replaced (SURVEY.md section 8(f) rank 4) over the batched C ABI:
`SignKeys::phase4`, `LocalSignature::{phase5_local_sig, phase5a_broadcast_5b_zkproof, phase5c, phase5d, output_signature}` of
/root/reference/src/protocols/multi_party_ecdsa/gg_2018/party_i.rs:455-730.  A batch is `sessions` signing sessions of `parties`
signers; element u = session * parties + party and every argument is a flat element-major sequence.  Phases 1-3 of GG18 are the
MtA of the hot path with an empty statement list (gg20.mta_message_a / mta_message_b / mta_get_alpha with n_st = 0) plus scalar
sums (Engine.scalar_op).  No arithmetic happens here — only packing."""
from __future__ import annotations

import ctypes
from typing import Sequence

import numpy as np

from . import HOST, Engine, ints_to_limbs, limbs_to_ints, _ptr
from .gg20 import _pts, unpack_point


def _bind(lib):
    if getattr(lib, "_gg18_bound", False):
        return
    V, S, I = ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int
    lib.tecdsa_gg18_phase4_batch.argtypes = [V, I] + [V] * 7 + [S, I]
    lib.tecdsa_gg18_local_sig_batch.argtypes = [V] * 6 + [S, I]
    lib.tecdsa_gg18_phase5a_batch.argtypes = [V] * 14 + [S, I]
    lib.tecdsa_gg18_phase5c_batch.argtypes = [V, I] + [V] * 14 + [S, I]
    lib.tecdsa_gg18_phase5d_batch.argtypes = [V, I] + [V] * 5 + [S, I]
    lib.tecdsa_gg18_output_signature_batch.argtypes = [V, I] + [V] * 8 + [S, I]
    lib._gg18_bound = True


def _points(a: np.ndarray):
    return [unpack_point(v) for v in limbs_to_ints(a)]


def phase4(eng: Engine, parties: int, delta_inv, b_proof_pk, g_gamma, blind, com):
    """`SignKeys::phase4` (party_i.rs:455-485).  b_proof_pk[u] = the `parties` DLogProof public keys element u holds (entry j from
    signer j; its own entry = its own g^gamma) -> (R per element, status)"""
    _bind(eng.lib)
    count = len(delta_inv)
    flat = [p for row in b_proof_pk for p in row]
    ins = [ints_to_limbs(delta_inv, 8), _pts(flat), _pts(g_gamma), ints_to_limbs(blind, 8), ints_to_limbs(com, 8)]
    R, st = np.zeros((count, 16), np.uint32), np.full(count, 255, np.uint8)
    eng._ck(eng.lib.tecdsa_gg18_phase4_batch(eng._ctx, parties, *[_ptr(a) for a in ins], _ptr(R), _ptr(st), count // parties, HOST), "gg18_phase4")
    return _points(R), st


def local_sig(eng: Engine, message, R, k_i, sigma_i):
    """`LocalSignature::phase5_local_sig` (party_i.rs:489-511): s_i = m k_i + r sigma_i"""
    _bind(eng.lib)
    count = len(k_i)
    ins = [ints_to_limbs(message, 8), _pts(R), ints_to_limbs(k_i, 8), ints_to_limbs(sigma_i, 8)]
    out = np.zeros((count, 8), np.uint32)
    eng._ck(eng.lib.tecdsa_gg18_local_sig_batch(eng._ctx, *[_ptr(a) for a in ins], _ptr(out), count, HOST), "gg18_local_sig")
    return limbs_to_ints(out)


def phase5a(eng: Engine, R, s_i, l_i, rho_i, blind, heg_s1, heg_s2, dlog_nonce):
    """`phase5a_broadcast_5b_zkproof` (party_i.rs:513-558) -> dict(com, decom[n][48] = V|A|B, heg[n][48], dlog[n][40], status)"""
    _bind(eng.lib)
    count = len(s_i)
    ins = [_pts(R)] + [ints_to_limbs(v, 8) for v in (s_i, l_i, rho_i, blind, heg_s1, heg_s2, dlog_nonce)]
    com, decom = np.zeros((count, 8), np.uint32), np.zeros((count, 48), np.uint32)
    heg, dlog = np.zeros((count, 48), np.uint32), np.zeros((count, 40), np.uint32)
    st = np.full(count, 255, np.uint8)
    eng._ck(eng.lib.tecdsa_gg18_phase5a_batch(eng._ctx, *[_ptr(a) for a in ins], _ptr(com), _ptr(decom), _ptr(heg), _ptr(dlog), _ptr(st), count, HOST),
            "gg18_phase5a")
    return {"com": com, "decom": decom, "heg": heg, "dlog": dlog, "status": st}


def phase5c(eng: Engine, parties: int, R, y, message, rho_i, l_i, blind2, com: np.ndarray, decom: np.ndarray, blind, heg: np.ndarray, dlog: np.ndarray):
    """`phase5c` (party_i.rs:560-629) -> dict(com2, decom2[n][32] = u_i|t_i, status)"""
    _bind(eng.lib)
    count = len(rho_i)
    ins = [_pts(R), _pts(y), ints_to_limbs(message, 8), ints_to_limbs(rho_i, 8), ints_to_limbs(l_i, 8), ints_to_limbs(blind2, 8),
           np.ascontiguousarray(com, np.uint32), np.ascontiguousarray(decom, np.uint32), ints_to_limbs(blind, 8),
           np.ascontiguousarray(heg, np.uint32), np.ascontiguousarray(dlog, np.uint32)]
    com2, decom2 = np.zeros((count, 8), np.uint32), np.zeros((count, 32), np.uint32)
    st = np.full(count, 255, np.uint8)
    eng._ck(eng.lib.tecdsa_gg18_phase5c_batch(eng._ctx, parties, *[_ptr(a) for a in ins], _ptr(com2), _ptr(decom2), _ptr(st), count // parties, HOST),
            "gg18_phase5c")
    return {"com2": com2, "decom2": decom2, "status": st}


def phase5d(eng: Engine, parties: int, decom2: np.ndarray, blind2, com2: np.ndarray, decom: np.ndarray) -> np.ndarray:
    """`phase5d` (party_i.rs:631-665) -> status (0 = Ok(s_i), 11 = InvalidCom, 2 = InvalidKey)"""
    _bind(eng.lib)
    count = decom2.shape[0]
    ins = [np.ascontiguousarray(decom2, np.uint32), ints_to_limbs(blind2, 8), np.ascontiguousarray(com2, np.uint32), np.ascontiguousarray(decom, np.uint32)]
    st = np.full(count, 255, np.uint8)
    eng._ck(eng.lib.tecdsa_gg18_phase5d_batch(eng._ctx, parties, *[_ptr(a) for a in ins], _ptr(st), count // parties, HOST), "gg18_phase5d")
    return st


def output_signature(eng: Engine, parties: int, R, y, message, s_i):
    """`output_signature` (party_i.rs:666-703) with the in-tree `verify` (:706-730) -> (r, s, recid, status) per element"""
    _bind(eng.lib)
    count = len(s_i)
    ins = [_pts(R), _pts(y), ints_to_limbs(message, 8), ints_to_limbs(s_i, 8)]
    r, s = np.zeros((count, 8), np.uint32), np.zeros((count, 8), np.uint32)
    rec, st = np.zeros(count, np.uint8), np.full(count, 255, np.uint8)
    eng._ck(eng.lib.tecdsa_gg18_output_signature_batch(eng._ctx, parties, *[_ptr(a) for a in ins], _ptr(r), _ptr(s), _ptr(rec), _ptr(st), count // parties, HOST),
            "gg18_output_signature")
    return limbs_to_ints(r), limbs_to_ints(s), rec, st


# ----------------------------------------------------------------------------- whole signing protocol over the batch calls
def sign_batch(eng: Engine, keys, parties: int, key_rows, w, y, message, rnd):
    """GG18 signing (gg_2018/test.rs `sign`: phases 1-5 + output_signature) for `sessions` sessions of `parties` signers, element
    u = session * parties + party, as a sequence of batch calls.  key_rows[u] = the element's Paillier key row in `keys`, w[u] its
    Lagrange-weighted share w_i = lambda_i x_i, y[u] the public key, message[u] the hashed message; rnd = dict of per-element
    lists k, gamma, blind (phase-1 commitment), r_a (MessageA randomness), l, rho, blind5, blind5c, heg_s1, heg_s2, dlog_nonce, and
    per ordered pair (alice u, bob v != u of the same session; pair index u * (parties - 1) + j) lists r_b_gamma, beta_tag_gamma,
    r_b_w, beta_tag_w, and the four DLogProof nonces nb_gamma, nbt_gamma, nb_w, nbt_w.
    -> dict(r, s, recid, status) per element; status is the first failing phase's code."""
    from . import gg20
    _bind(eng.lib)
    U = len(key_rows)
    P1 = parties - 1
    k, gamma = list(rnd["k"]), list(rnd["gamma"])
    status = np.zeros(U, np.uint8)

    def first_fail(st, idx=None):
        for t, code in enumerate(st):
            u = t if idx is None else idx[t]
            if code and not status[u]:
                status[u] = code

    # phase 1: commit to g^gamma, MessageA = Enc_i(k_i) (no range proofs in GG18: MessageA::a(&k_i, &ek, &[]))
    g_gamma = eng.secp_mul(None, gamma)
    com = gg20.hash_commitment(eng, g_gamma, rnd["blind"])
    c_a, _ = gg20.mta_message_a(eng, keys, list(key_rows), [[] for _ in range(U)], k, rnd["r_a"], [[] for _ in range(U)])
    # phase 2: every ordered pair runs MtA twice (b = gamma_j and b = w_j) under Alice's key
    alice = [u for u in range(U) for _ in range(P1)]
    bob = [u // parties * parties + (j if j < u % parties else j + 1) for u in range(U) for j in range(P1)]
    none = [[] for _ in alice]
    empty = {f: none for f in ("z", "e", "s", "s1", "s2")}
    a_rows, a_ca = [key_rows[u] for u in alice], [c_a[u] for u in alice]
    cb_g, bp_g, btp_g, beta_g, st = gg20.mta_message_b(eng, keys, a_rows, none, [gamma[v] for v in bob], a_ca, empty, rnd["r_b_gamma"], rnd["beta_tag_gamma"],
                                                        rnd["nb_gamma"], rnd["nbt_gamma"])
    first_fail(st, bob)
    cb_w, bp_w, btp_w, beta_w, st = gg20.mta_message_b(eng, keys, a_rows, none, [w[v] for v in bob], a_ca, empty, rnd["r_b_w"], rnd["beta_tag_w"],
                                                        rnd["nb_w"], rnd["nbt_w"])
    first_fail(st, bob)
    alpha_g, _, st = gg20.mta_get_alpha(eng, keys, a_rows, [k[u] for u in alice], cb_g, bp_g, btp_g)
    first_fail(st, alice)
    alpha_w, _, st = gg20.mta_get_alpha(eng, keys, a_rows, [k[u] for u in alice], cb_w, bp_w, btp_w)
    first_fail(st, alice)
    # delta_i = k_i gamma_i + sum_j alpha_ij + sum_j beta_ji ; sigma_i likewise with w (party_i.rs:427-445)
    delta = eng.scalar_op("mul", k, gamma)
    sigma = eng.scalar_op("mul", k, w)
    for j in range(P1):
        delta = eng.scalar_op("add", delta, [alpha_g[u * P1 + j] for u in range(U)])
        sigma = eng.scalar_op("add", sigma, [alpha_w[u * P1 + j] for u in range(U)])
    as_bob = {v: [] for v in range(U)}
    for t, v in enumerate(bob):
        as_bob[v].append(t)
    for j in range(P1):
        delta = eng.scalar_op("add", delta, [beta_g[as_bob[v][j]] for v in range(U)])
        sigma = eng.scalar_op("add", sigma, [beta_w[as_bob[v][j]] for v in range(U)])
    # phase 3: delta^-1 of the session sum
    tot = [0] * U
    for j in range(parties):
        tot = eng.scalar_op("add", tot, [delta[u // parties * parties + j] for u in range(U)])
    dinv = eng.scalar_op("inv", tot)
    for u in range(U):
        if dinv[u] is None and not status[u]:
            status[u] = 4
    dinv = [d or 0 for d in dinv]
    # phase 4: R; the public key of the MessageB proof element u received from signer v is g^gamma_v as v proved it
    pk_of = {}
    for t, (u, v) in enumerate(zip(alice, bob)):
        pk_of[(u, v)] = unpack_point(limbs_to_ints(bp_g[t:t + 1, :16])[0])
    pks = [[g_gamma[u] if (u // parties * parties + j) == u else pk_of[(u, u // parties * parties + j)] for j in range(parties)] for u in range(U)]
    R, st = phase4(eng, parties, dinv, pks, g_gamma, rnd["blind"], com)
    first_fail(st)
    Rs = [p if p is not None else (0, 0) for p in R]
    # phase 5
    s_i = local_sig(eng, message, Rs, k, sigma)
    a5 = phase5a(eng, Rs, s_i, rnd["l"], rnd["rho"], rnd["blind5"], rnd["heg_s1"], rnd["heg_s2"], rnd["dlog_nonce"])
    first_fail(a5["status"])
    c5 = phase5c(eng, parties, Rs, y, message, rnd["rho"], rnd["l"], rnd["blind5c"], a5["com"], a5["decom"], rnd["blind5"], a5["heg"], a5["dlog"])
    first_fail(c5["status"])
    first_fail(phase5d(eng, parties, c5["decom2"], rnd["blind5c"], c5["com2"], a5["decom"]))
    r, s, rec, st = output_signature(eng, parties, Rs, y, message, s_i)
    first_fail(st)
    return {"r": r, "s": s, "recid": rec, "status": status, "R": R, "s_i": s_i}


# ----------------------------------------------------------------------------- key generation (gg_2018/party_i.rs:155-317)
def keygen_batch(eng: Engine, t: int, n: int, u, p_q, blind, polynomials, dlog_nonce):
    """GG18 key generation for `sessions` groups of n parties (element e = session * n + party) as batch calls:
    `Keys::phase1_broadcast_phase3_proof_of_correct_key`, `phase1_verify_com_phase3_verify_correct_key_phase2_distribute`,
    `phase2_verify_vss_construct_keypair_phase3_pok_dlog`, `verify_dlog_proofs`.  u[e] = the party's secret u_i, p_q[e] its Paillier
    primes, blind[e] the commitment blinding factor, polynomials[e] = [u_i, a_1 .. a_t] (the coefficients `VerifiableSS::share`
    samples), dlog_nonce[e] the nonce of the final DLogProof.
    -> dict(status per element (0 / 2 = InvalidKey / 12 = InvalidSS), y per element (the group key), x_i (secret share), y_i, com,
            correct_key_proof, vss commitments, shares, dlog proofs)"""
    from . import gg20, keygen
    E = len(u)
    assert E % n == 0 and all(poly[0] == ui for poly, ui in zip(polynomials, u))
    sess = lambda e: e // n * n
    status = np.zeros(E, np.uint8)
    # phase 1: y_i, commitment, NiCorrectKeyProof
    y_i = eng.secp_mul(None, list(u))
    com = gg20.hash_commitment(eng, y_i, blind)
    n_list = [p * q for p, q in p_q]
    sigma, st = keygen.correct_key_prove(eng, p_q)
    # phase 1 verification by every receiver = one check per sender (the same for all receivers), then phase 2 distribution
    reopen = gg20.hash_commitment(eng, y_i, blind)
    ck = keygen.correct_key_verify(eng, n_list, sigma)
    bad_sender = [reopen[e] != com[e] or ck[e] != 0 or st[e] != 0 for e in range(E)]
    for e in range(E):
        if any(bad_sender[sess(e):sess(e) + n]):
            status[e] = 2                                         # Err(InvalidKey)
    shares, commitments = keygen.vss_share(eng, t, n, polynomials)
    # phase 2: receiver r validates the share of every sender s of its group: pairs (r, s)
    recv = [r for r in range(E) for _ in range(n)]
    send = [sess(r) + j for r in range(E) for j in range(n)]
    ok = keygen.vss_validate_share(eng, [commitments[s] for s in send], [shares[s][r % n] for r, s in zip(recv, send)], [r % n + 1 for r in recv])
    for i, (r, s) in enumerate(zip(recv, send)):
        if (ok[i] != 0 or commitments[s][0] != y_i[s]) and not status[r]:
            status[r] = 12                                        # Err(InvalidSS)
    y = [y_i[sess(e)] for e in range(E)]
    x_i = [shares[sess(e)][e % n] for e in range(E)]
    for j in range(1, n):
        y = eng.point_add(y, [y_i[sess(e) + j] for e in range(E)])
        x_i = eng.scalar_op("add", x_i, [shares[sess(e) + j][e % n] for e in range(E)])
    dlog = gg20.dlog_prove(eng, x_i, dlog_nonce)
    dv = gg20.dlog_verify(eng, dlog)
    for e in range(E):
        if dv[sess(e):sess(e) + n].any() and not status[e]:
            status[e] = 2                                         # verify_dlog_proofs -> Err(InvalidKey)
    return {"status": status, "y": y, "x_i": x_i, "y_i": y_i, "com": com, "correct_key_proof": sigma, "commitments": commitments, "shares": shares, "dlog": dlog}


# ----------------------------------------------------------------------------- signing as one call (tecdsa_gg18_signing_batch)
# widths (limbs) of the inputs: per element ([E][w]) and per pair ([signers-1][E][w], slab j = element u towards its j-th peer)
ELEMENT_FIELDS = {"k": 8, "gamma": 8, "blind": 8, "r_a": 64, "l": 8, "rho": 8, "blind5": 8, "blind5c": 8, "heg_s1": 8, "heg_s2": 8, "dlog_nonce": 8}
PAIR_FIELDS = {"beta_tag_gamma": 64, "r_gamma": 64, "beta_tag_w": 64, "r_w": 64, "nonce_gamma_b": 8, "nonce_gamma_beta": 8, "nonce_w_b": 8, "nonce_w_beta": 8}
IN_FIELDS = list(ELEMENT_FIELDS) + list(PAIR_FIELDS)
OUT_FIELDS = ("status", "R", "sig_r", "sig_s", "recid", "complete")
# TECDSA_RNDS_G18_*: one stream per field, in the order of tecdsa_gg18_signing_in
RNDS = {f: 80 + i for i, f in enumerate(IN_FIELDS)}


class _SigningIn(ctypes.Structure):
    _fields_ = [(n, ctypes.c_void_p) for n in IN_FIELDS]


class _SigningOut(ctypes.Structure):
    _fields_ = [(n, ctypes.c_void_p) for n in OUT_FIELDS]


def _descriptors(sessions, signers: int) -> np.ndarray:
    """[n][1 + signers] uint32 on the host (a CUDA tensor is copied back: the descriptors are public)"""
    from .keygen import _host
    return np.ascontiguousarray(_host(sessions) if not isinstance(sessions, (list, tuple)) else np.asarray(sessions), dtype=np.uint32).reshape(-1, 1 + signers)


def sample_inputs(eng: Engine, keys, signers: int, sessions, seed=None, mem: int = HOST):
    """Every input of `sign_device`, drawn by `tecdsa_sample_batch` as the reference draws it (kinds in tecdsa_gg18_signing_in) on
    the TECDSA_RNDS_G18_* streams.  Element u = session * signers + position has element id (sub << 32) | u, sub = 0 for the
    per-element fields and the peer index j for the per-pair fields (the rule of the key-generation streams).  keys = gg20.KeySets;
    sessions = [n][1 + signers] (key set, then s_l[p] - 1).  -> dict field -> array in the layout of tecdsa_gg18_signing_in (numpy
    for HOST; CUDA tensors for DEVICE, which never reach the host).  seed=None draws a fresh seed; a seed serves ONE call."""
    from . import SAMPLE_BELOW, SAMPLE_BITS, SAMPLE_SCALAR, EngineError, gg20, seed_words, ints_to_limbs
    from .keygen import _buffer, _host, _upload
    lib = eng.lib
    if not getattr(lib, "_sample_bound", False):
        V, S_, I_ = ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int
        lib.tecdsa_sample_batch.argtypes = [V, V, ctypes.c_uint64, ctypes.c_uint32, I_, I_, V, V, S_, I_, V, V, S_, I_]
        lib._sample_bound = True
    d = _descriptors(sessions, signers)
    T, P, n = signers, keys.parties, d.shape[0]
    E = n * T
    N = _upload(ints_to_limbs(keys.table(0, 64), 64), mem, eng.device)         # the Paillier N of every key row
    own = (d[:, :1] * P + d[:, 1:]).reshape(E).astype(np.uint32)
    pos = np.arange(E) % T
    base = np.arange(E) - pos
    sw = seed_words(gg20.fresh_seed(seed))

    def draw(out, name, kind, sub=0, rows=None, bits=0):
        st = _buffer((E,), np.uint8, mem, eng.device)
        ix = None if rows is None else _upload(rows, mem, eng.device)
        eng._ck(lib.tecdsa_sample_batch(eng._ctx, _ptr(sw), sub << 32, RNDS[name], kind, bits, _ptr(N) if rows is not None else None, _ptr(ix),
                                        0 if rows is None else N.shape[0], out.shape[-1], _ptr(out), _ptr(st), E, mem), "sample_batch")
        bad = np.flatnonzero(_host(st))
        if bad.size:
            raise EngineError(f"sampling {name}: element {int(bad[0])} has status {int(_host(st)[bad[0]])}")

    inp = {f: _buffer((E, w), np.uint32, mem, eng.device) for f, w in ELEMENT_FIELDS.items()}
    inp.update({f: _buffer((T - 1, E, w), np.uint32, mem, eng.device) for f, w in PAIR_FIELDS.items()})
    try:
        for f in ("k", "gamma", "l", "rho", "heg_s1", "heg_s2", "dlog_nonce"):
            draw(inp[f], f, SAMPLE_SCALAR)
        for f in ("blind", "blind5", "blind5c"):
            draw(inp[f], f, SAMPLE_BITS, bits=256)
        draw(inp["r_a"], "r_a", SAMPLE_BELOW, rows=own)
        for j in range(T - 1):
            peer = own[base + np.where(j < pos, j, j + 1)].astype(np.uint32)
            for f in ("beta_tag_gamma", "r_gamma", "beta_tag_w", "r_w"):
                draw(inp[f][j], f, SAMPLE_BELOW, j, rows=peer)
            for f in ("nonce_gamma_b", "nonce_gamma_beta", "nonce_w_b", "nonce_w_beta"):
                draw(inp[f][j], f, SAMPLE_SCALAR, j)
    finally:
        sw[:] = 0
    return inp


def sign_device(eng: Engine, keys, signers: int, sessions, message, inp, mem: int = HOST, out=None, check: bool = True):
    """GG18 signing (gg_2018/test.rs `sign`: phases 1-5, output_signature, verify) for every session as ONE call
    (tecdsa_gg18_signing_batch).  sessions = [n][1 + signers]; message = [n] ints (reduced mod q) or an [n][8] limb array;
    inp = the dict `sample_inputs` returns (or the same fields from elsewhere).  -> dict(status [E], R [E][16], r [n][8], s [n][8],
    recid [n], complete [n]): numpy arrays for HOST, CUDA tensors for DEVICE (the caller's, when `out` holds them under the names
    of tecdsa_gg18_signing_out; sessions and message are then CUDA tensors too).  A session that did not complete has zero R and
    signature.  check=False returns the call's rc instead of raising."""
    from .keygen import _buffer
    lib = eng.lib
    if not getattr(lib, "_gg18_signing_bound", False):
        V = ctypes.c_void_p
        lib.tecdsa_gg18_signing_batch.argtypes = [V, V, ctypes.c_int, ctypes.c_size_t, ctypes.c_int, V, V, ctypes.POINTER(_SigningIn),
                                                  ctypes.POINTER(_SigningOut)]
        lib._gg18_signing_bound = True
    if isinstance(message, (list, tuple)):
        message = ints_to_limbs([int(m) for m in message], 8)
    if mem == HOST:
        sessions = _descriptors(sessions, signers)
        inp = {f: None if v is None else np.ascontiguousarray(v, dtype=np.uint32) for f, v in inp.items()}
        message = np.ascontiguousarray(message, dtype=np.uint32)
    n = sessions.shape[0]
    E = n * signers
    if out is None:
        out = {"status": _buffer((E,), np.uint8, mem, eng.device), "R": _buffer((E, 16), np.uint32, mem, eng.device),
               "sig_r": _buffer((n, 8), np.uint32, mem, eng.device), "sig_s": _buffer((n, 8), np.uint32, mem, eng.device),
               "recid": _buffer((n,), np.uint8, mem, eng.device), "complete": _buffer((n,), np.uint8, mem, eng.device)}
    si = _SigningIn(*[_ptr(inp[f]) for f in IN_FIELDS])
    so = _SigningOut(*[_ptr(out[f]) for f in OUT_FIELDS])
    rc = lib.tecdsa_gg18_signing_batch(eng._ctx, keys.handle, signers, n, mem, _ptr(sessions), _ptr(message), ctypes.byref(si), ctypes.byref(so))
    if not check:
        return rc
    eng._ck(rc, "gg18_signing_batch")
    return {"status": out["status"], "R": out["R"], "r": out["sig_r"], "s": out["sig_s"], "recid": out["recid"], "complete": out["complete"]}
