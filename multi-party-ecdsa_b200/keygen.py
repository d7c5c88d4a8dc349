"""Host-side mirror of the key-generation path (SURVEY.md section 8(f) rank 1), batched through the C ABI:
`NiCorrectKeyProof::{proof,verify}`, `CompositeDLogProof::{prove,verify}`, `VerifiableSS::{share,validate_share}`,
`generate_h1_h2_N_tilde` and the per-phase checks of `Keys` as called from
/root/reference/src/protocols/multi_party_ecdsa/gg_2020/party_i.rs:137-156,219-438.  No arithmetic happens here: the functions
pack limbs, call the library and combine status bytes."""
from __future__ import annotations

import ctypes
from dataclasses import dataclass
from typing import List, Optional, Sequence, Tuple

import numpy as np

from . import HOST, Engine, ints_to_limbs, _ptr
from . import limbs_to_ints
from .gg20 import pack_point, unpack_point
from .wire import DecryptionKey, DLogStatement, EncryptionKey, LoadedLocalKey

SALT_STRING = bytes([75, 90, 101, 110])            # zk-paillier `SALT_STRING` [R]


def _bind(lib):
    if getattr(lib, "_keygen_bound", False):
        return
    V, S, I = ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int
    lib.tecdsa_correct_key_verify_batch.argtypes = [V, V, V, V, I, V, S, I]
    lib.tecdsa_composite_dlog_verify_batch.argtypes = [V, V, V, V, V, V, I, V, S, I]
    lib.tecdsa_vss_validate_share_batch.argtypes = [V, V, I, V, V, V, S, I]
    lib.tecdsa_correct_key_prove_batch.argtypes = [V, V, V, V, I, V, V, S, I]
    lib.tecdsa_composite_dlog_prove_batch.argtypes = [V, V, V, V, V, I, V, V, V, I, S, I]
    lib.tecdsa_vss_share_batch.argtypes = [V, I, I, V, V, V, S, I]
    lib.tecdsa_h1_h2_n_tilde_batch.argtypes = [V] * 10 + [S, I]
    lib._keygen_bound = True


def correct_key_verify(eng: Engine, n_list: Sequence[int], sigma_vecs: Sequence[Sequence[int]], salt: bytes = SALT_STRING) -> np.ndarray:
    """-> status[count] (0 = accept).  sigma_vecs[i] are the 11 values of proof i; any other length rejects on the host."""
    _bind(eng.lib)
    count = len(n_list)
    N = ints_to_limbs(n_list, 64)
    flat, short = [], np.zeros(count, dtype=bool)
    for i, sv in enumerate(sigma_vecs):
        if len(sv) != 11 or any(s < 0 or s >> 2048 for s in sv):
            short[i] = True
            sv = [0] * 11
        flat += list(sv)
    Sg = ints_to_limbs(flat, 64)
    st = np.full(count, 255, dtype=np.uint8)
    salt_arr = np.frombuffer(salt, dtype=np.uint8).copy() if salt else None
    eng._ck(eng.lib.tecdsa_correct_key_verify_batch(eng._ctx, _ptr(N), _ptr(Sg), _ptr(salt_arr) if salt_arr is not None else None, len(salt),
                                                    _ptr(st), count, HOST), "correct_key_verify")
    st[short] = 10                                   # TECDSA_ST_PROOF
    return st


def composite_dlog_verify(eng: Engine, statements: Sequence[Tuple[int, int, int]], proofs: Sequence[Tuple[int, int]], y_limbs: int = 92) -> np.ndarray:
    """statements[i] = (N, g, ni), proofs[i] = (x, y) -> status[count]"""
    _bind(eng.lib)
    count = len(statements)
    N = ints_to_limbs([s[0] for s in statements], 64)
    G = ints_to_limbs([s[1] % (1 << 2048) for s in statements], 64)
    NI = ints_to_limbs([s[2] % (1 << 2048) for s in statements], 64)
    bad = np.array([p[1] < 0 or p[1] >> (32 * y_limbs) != 0 or p[0] < 0 or p[0] >> 2048 != 0 for p in proofs], dtype=bool)
    X = ints_to_limbs([0 if b else p[0] for p, b in zip(proofs, bad)], 64)
    Y = ints_to_limbs([0 if b else p[1] for p, b in zip(proofs, bad)], y_limbs)
    st = np.full(count, 255, dtype=np.uint8)
    eng._ck(eng.lib.tecdsa_composite_dlog_verify_batch(eng._ctx, _ptr(N), _ptr(G), _ptr(NI), _ptr(X), _ptr(Y), y_limbs, _ptr(st), count, HOST),
            "composite_dlog_verify")
    st[bad] = 10
    return st


def vss_validate_share(eng: Engine, commitments: Sequence[Sequence], shares: Sequence[int], indices: Sequence[int]) -> np.ndarray:
    """commitments[i] = the t+1 coefficient commitments (oracle points) of scheme i -> status[count]"""
    _bind(eng.lib)
    count = len(shares)
    nc = len(commitments[0])
    assert all(len(c) == nc for c in commitments)
    C = ints_to_limbs([pack_point(p) for cs in commitments for p in cs], 16)
    Sh = ints_to_limbs([s % (1 << 256) for s in shares], 8)
    idx = np.asarray(indices, dtype=np.uint32)
    st = np.full(count, 255, dtype=np.uint8)
    eng._ck(eng.lib.tecdsa_vss_validate_share_batch(eng._ctx, _ptr(C), nc, _ptr(Sh), _ptr(idx), _ptr(st), count, HOST), "vss_validate_share")
    return st


# ----------------------------------------------------------------------------- prove side
def correct_key_prove(eng: Engine, pq: Sequence[Tuple[int, int]], salt: bytes = SALT_STRING):
    """`NiCorrectKeyProof::proof(&dk, None)` batched: pq[i] = (p, q) -> (list of 11-element sigma vectors, status)"""
    _bind(eng.lib)
    count = len(pq)
    P, Qv = ints_to_limbs([x[0] for x in pq], 32), ints_to_limbs([x[1] for x in pq], 32)
    sig = np.zeros((count * 11, 64), dtype=np.uint32)
    st = np.full(count, 255, dtype=np.uint8)
    salt_arr = np.frombuffer(salt, dtype=np.uint8).copy() if salt else None
    eng._ck(eng.lib.tecdsa_correct_key_prove_batch(eng._ctx, _ptr(P), _ptr(Qv), _ptr(salt_arr) if salt_arr is not None else None, len(salt),
                                                   _ptr(sig), _ptr(st), count, HOST), "correct_key_prove")
    flat = limbs_to_ints(sig)
    return [flat[11 * i:11 * i + 11] for i in range(count)], st


def composite_dlog_prove(eng: Engine, statements: Sequence[Tuple[int, int, int]], secrets: Sequence[int], nonces: Sequence[int],
                         secret_limbs: int = 64, y_limbs: int = 76):
    """`CompositeDLogProof::prove(&DLogStatement{N, g, ni}, &secret)` with the sampled nonce explicit -> list of (x, y)"""
    _bind(eng.lib)
    count = len(statements)
    N, G, NI = (ints_to_limbs([s[k] for s in statements], 64) for k in range(3))
    Sec, R = ints_to_limbs(secrets, secret_limbs), ints_to_limbs(nonces, 16)
    X, Y = np.zeros((count, 64), dtype=np.uint32), np.zeros((count, y_limbs), dtype=np.uint32)
    eng._ck(eng.lib.tecdsa_composite_dlog_prove_batch(eng._ctx, _ptr(N), _ptr(G), _ptr(NI), _ptr(Sec), secret_limbs, _ptr(R), _ptr(X), _ptr(Y), y_limbs,
                                                      count, HOST), "composite_dlog_prove")
    return list(zip(limbs_to_ints(X), limbs_to_ints(Y)))


def vss_share(eng: Engine, t: int, n: int, polynomials: Sequence[Sequence[int]]):
    """`VerifiableSS::share(t, n, &secret)` with explicit coefficients (polynomials[i][0] = the secret) ->
    (shares[i] = [f(1)..f(n)], commitments[i] = [(x, y) of a_j*G])"""
    _bind(eng.lib)
    count = len(polynomials)
    assert all(len(p) == t + 1 for p in polynomials)
    C = ints_to_limbs([c for p in polynomials for c in p], 8)
    Sh, Cm = np.zeros((count * n, 8), dtype=np.uint32), np.zeros((count * (t + 1), 16), dtype=np.uint32)
    eng._ck(eng.lib.tecdsa_vss_share_batch(eng._ctx, t, n, _ptr(C), _ptr(Sh), _ptr(Cm), count, HOST), "vss_share")
    sh, cm = limbs_to_ints(Sh), [unpack_point(v) for v in limbs_to_ints(Cm)]
    return [sh[i * n:(i + 1) * n] for i in range(count)], [cm[i * (t + 1):(i + 1) * (t + 1)] for i in range(count)]


def h1_h2_n_tilde(eng: Engine, setups: Sequence[Tuple[int, int, int, int]]):
    """`generate_h1_h2_N_tilde` with explicit samples: setups[i] = (p~, q~, h1, xhi) -> ([(N~, h1, h2, phi - xhi, phi - xhi^-1)], status)"""
    _bind(eng.lib)
    count = len(setups)
    P, Qv = ints_to_limbs([s[0] for s in setups], 32), ints_to_limbs([s[1] for s in setups], 32)
    H1, X = ints_to_limbs([s[2] for s in setups], 64), ints_to_limbs([s[3] for s in setups], 64)
    outs = [np.zeros((count, 64), dtype=np.uint32) for _ in range(4)]
    st = np.full(count, 255, dtype=np.uint8)
    eng._ck(eng.lib.tecdsa_h1_h2_n_tilde_batch(eng._ctx, _ptr(P), _ptr(Qv), _ptr(H1), _ptr(X), *[_ptr(o) for o in outs], _ptr(st), count, HOST), "h1_h2_n_tilde")
    nt, h2, xn, xin = (limbs_to_ints(o) for o in outs)
    return [(nt[i], setups[i][2], h2[i], xn[i], xin[i]) for i in range(count)], st


# ----------------------------------------------------------------------------- per-phase checks of `Keys` (batched over messages)
def phase1_verify(eng: Engine, broadcasts: Sequence, decommits: Sequence) -> np.ndarray:
    """The per-sender term of `phase1_verify_com_phase3_verify_correct_key_verify_dlog_phase2_distribute` (party_i.rs:272-305) for a
    batch of (KeyGenBroadcastMessage1, KeyGenDecommitMessage1) pairs (duck-typed like oracle.keygen_oracle's dataclasses):
    commitment opens, NiCorrectKeyProof verifies, both moduli are 2047..2048 bits, both CompositeDLogProofs verify.
    -> bool[count] (False = that sender is a `bad_actor`)."""
    from .gg20 import hash_commitment
    count = len(broadcasts)
    ok = np.ones(count, dtype=bool)
    com = hash_commitment(eng, [d.y_i for d in decommits], [d.blind_factor for d in decommits])
    ok &= np.array([c == b.com for c, b in zip(com, broadcasts)])
    ok &= correct_key_verify(eng, [b.e.n for b in broadcasts], [b.correct_key_proof for b in broadcasts]) == 0
    ok &= np.array([2047 <= b.e.n.bit_length() <= 2048 and 2047 <= b.dlog_statement.N.bit_length() <= 2048 for b in broadcasts])
    st1 = [(b.dlog_statement.N, b.dlog_statement.g, b.dlog_statement.ni) for b in broadcasts]
    st2 = [(b.dlog_statement.N, b.dlog_statement.ni, b.dlog_statement.g) for b in broadcasts]
    pf = [(b.composite_dlog_proof_base_h1.x, b.composite_dlog_proof_base_h1.y) for b in broadcasts] + \
         [(b.composite_dlog_proof_base_h2.x, b.composite_dlog_proof_base_h2.y) for b in broadcasts]
    cd = composite_dlog_verify(eng, st1 + st2, pf) == 0
    return ok & cd[:count] & cd[count:]


def phase2_verify_vss(eng: Engine, y_vec: Sequence, shares_for_me: Sequence[int], vss_vec: Sequence, index: int) -> np.ndarray:
    """The per-sender term of `phase2_verify_vss_construct_keypair_phase3_pok_dlog` (party_i.rs:334-349): validate_share and
    commitments[0] == y_i.  -> bool[count]"""
    ok = vss_validate_share(eng, [v.commitments for v in vss_vec], shares_for_me, [index] * len(shares_for_me)) == 0
    return ok & np.array([v.commitments[0] == y for v, y in zip(vss_vec, y_vec)])


# ----------------------------------------------------------------------------- GG20 key generation as one call
RNDS_KG_U, RNDS_KG_COEFF, RNDS_KG_BLIND, RNDS_KG_H1, RNDS_KG_XHI, RNDS_KG_CDL, RNDS_KG_DLOG = range(64, 71)     # TECDSA_RNDS_KG_*
CDL_NONCE_BITS = 512                              # zk-paillier CompositeDLogProof nonce bound [R]
# the input record of tecdsa_gg20_keygen_batch: field -> (limbs per row, rows per element); coeffs has t rows, one per a_k
RECORD = {"u": (8, 1), "coeffs": (8, None), "blind": (8, 1), "h1": (64, 1), "xhi": (64, 1), "cdl_nonce": (16, 2), "dlog_nonce": (8, 1)}


class _KeygenIn(ctypes.Structure):
    _fields_ = [(f, ctypes.c_void_p) for f in ("paillier_p", "paillier_q", "n_tilde_p", "n_tilde_q", "u", "coeffs", "blind", "h1", "xhi",
                                                "cdl_nonce", "dlog_nonce")]


class _KeygenOut(ctypes.Structure):
    _fields_ = [(f, ctypes.c_void_p) for f in ("x_i", "vss", "n", "dlog_st", "y", "pk", "status", "bad_actors", "complete")]


def _buffer(shape, dtype, mem, device):
    if mem == HOST:
        return np.zeros(shape, dtype=dtype)
    import torch
    tdt = {np.uint8: torch.uint8, np.uint32: torch.int32, np.uint64: torch.int64}[dtype]
    return torch.zeros(shape, dtype=tdt, device=f"cuda:{device}")


def _upload(a: np.ndarray, mem, device):
    if mem == HOST:
        return np.ascontiguousarray(a)
    import torch
    return torch.from_numpy(np.ascontiguousarray(a).view(np.int32)).to(f"cuda:{device}")


def _host(a) -> np.ndarray:
    if isinstance(a, np.ndarray):
        return a
    import torch
    a = a.cpu().numpy()
    return a.view({np.dtype(np.int32): np.uint32, np.dtype(np.int64): np.uint64}.get(a.dtype, a.dtype))


def sample_randomness(eng: Engine, t: int, n: int, n_tilde_primes: Sequence[Tuple[int, int]], seed: bytes, first_id: int = 0, mem: int = HOST):
    """Every input of `keygen_batch` except the primes, drawn by `tecdsa_sample_batch` as the reference draws it inside `Keys::create`,
    `phase1_broadcast_phase3_proof_of_correct_key_proof_of_correct_h1h2`, `VerifiableSS::share` and `DLogProof::prove`
    (gg_2020/party_i.rs:137-367): u_i, a_1..a_t and the DLog nonce SCALAR, blind BITS(256), h1 BELOW(N~), xhi UNIT(phi(N~)), the two
    CompositeDLog nonces BITS(512).  n_tilde_primes[e] = (p~, q~) of element e (len = groups * n).  Stream TECDSA_RNDS_KG_*, element
    id (sub << 32) + first_id + e (sub = k - 1 for a_k, 0 / 1 for the nonces of bases h1 / h2, else 0), so a batch split by first_id
    draws the same values.  -> dict field -> array in the layouts of RECORD (numpy for HOST; CUDA tensors for DEVICE, which never
    reach the host).  A (seed, first_id + e) pair must never be used twice."""
    from . import SAMPLE_BELOW, SAMPLE_BITS, SAMPLE_SCALAR, SAMPLE_UNIT, EngineError, seed_words
    lib = eng.lib
    if not getattr(lib, "_sample_bound", False):
        V, S, I = ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int
        lib.tecdsa_sample_batch.argtypes = [V, V, ctypes.c_uint64, ctypes.c_uint32, I, I, V, V, S, I, V, V, S, I]
        lib._sample_bound = True
    E = len(n_tilde_primes)
    if E % n or not 1 <= t <= n - 1:
        raise ValueError("keygen sampling: len(n_tilde_primes) must be a multiple of n, and 1 <= t <= n - 1")
    nt = _upload(ints_to_limbs([p * q for p, q in n_tilde_primes], 64), mem, eng.device)
    phi = _upload(ints_to_limbs([(p - 1) * (q - 1) for p, q in n_tilde_primes], 64), mem, eng.device)
    sw = seed_words(seed)

    def draw(name, kind, stream, limbs, sub=0, bound=None, bits=0):
        out, st = _buffer((E, limbs), np.uint32, mem, eng.device), _buffer((E,), np.uint8, mem, eng.device)
        eng._ck(lib.tecdsa_sample_batch(eng._ctx, _ptr(sw), (sub << 32) + first_id, stream, kind, bits, _ptr(bound), None, 0 if bound is None else E,
                                        limbs, _ptr(out), _ptr(st), E, mem), "sample_batch")
        bad = np.flatnonzero(_host(st))
        if bad.size:
            raise EngineError(f"keygen sampling {name}: element {int(bad[0])} could not be drawn")
        return out

    try:
        rec = {"u": draw("u", SAMPLE_SCALAR, RNDS_KG_U, 8), "blind": draw("blind", SAMPLE_BITS, RNDS_KG_BLIND, 8, bits=256),
               "h1": draw("h1", SAMPLE_BELOW, RNDS_KG_H1, 64, bound=nt), "xhi": draw("xhi", SAMPLE_UNIT, RNDS_KG_XHI, 64, bound=phi),
               "dlog_nonce": draw("dlog_nonce", SAMPLE_SCALAR, RNDS_KG_DLOG, 8)}
        coeffs = [draw("coeffs", SAMPLE_SCALAR, RNDS_KG_COEFF, 8, sub=k) for k in range(t)]
        cdl = [draw("cdl_nonce", SAMPLE_BITS, RNDS_KG_CDL, 16, sub=k, bits=CDL_NONCE_BITS) for k in range(2)]
    finally:
        sw[:] = 0
    if mem == HOST:
        rec["coeffs"], rec["cdl_nonce"] = np.stack(coeffs, axis=1), np.stack(cdl, axis=1)
    else:
        import torch
        rec["coeffs"], rec["cdl_nonce"] = torch.stack(coeffs, dim=1).contiguous(), torch.stack(cdl, dim=1).contiguous()
    return rec


def pack_randomness(t: int, rnd: Sequence[dict]) -> dict:
    """Per-element dicts of Python ints (u, coeffs = [a_1..a_t], blind, h1, xhi, cdl_nonce = (r1, r2), dlog_nonce) -> the HOST record"""
    rec = {f: ints_to_limbs([x for r in rnd for x in (r[f] if isinstance(r[f], (list, tuple)) else [r[f]])], limbs)
           for f, (limbs, _) in RECORD.items()}
    E = len(rnd)
    rec["coeffs"] = rec["coeffs"].reshape(E, t, 8)
    rec["cdl_nonce"] = rec["cdl_nonce"].reshape(E, 2, 16)
    return rec


@dataclass
class KeygenResult:
    status: np.ndarray              # [E] TECDSA_ST_* of each element
    bad_actors: np.ndarray          # [E] uint64, bit j = party j + 1
    complete: np.ndarray            # [groups] 1 = the group holds its LocalKeys
    keys: Optional[List[Optional[LoadedLocalKey]]]      # per element (None in an incomplete group); HOST only
    out: dict                       # the raw outputs of tecdsa_gg20_keygen_batch (numpy for HOST, CUDA tensors for DEVICE)


def keygen_batch(eng: Engine, t: int, n: int, paillier_primes: Sequence[Tuple[int, int]], n_tilde_primes: Sequence[Tuple[int, int]], rnd: dict,
                 mem: int = HOST) -> KeygenResult:
    """GG20 `Keygen` Round0..Round4 (gg_2020/state_machine/keygen/rounds.rs:26-300) for groups of n parties in ONE device call
    (tecdsa_gg20_keygen_batch).  Element e = g * n + (i - 1) is party i of group g; paillier_primes[e] = (p, q), n_tilde_primes[e] =
    (p~, q~); rnd = the record of `sample_randomness` / `pack_randomness` (on the device for DEVICE).  keys[e] has the fields of
    `LocalKey` (those of oracle.LocalKey plus its own VSS commitments) and feeds gg20.KeySets, gg20_general.offline_batch and
    wire.local_key as it is.  With DEVICE the outputs stay in `out` on the device and no key object is built."""
    E = len(paillier_primes)
    if len(n_tilde_primes) != E or E % n:
        raise ValueError("keygen_batch: one (p, q) and one (p~, q~) per element, groups * n elements")
    groups, dev = E // n, eng.device
    lib = eng.lib
    if not getattr(lib, "_gg20_keygen_bound", False):
        lib.tecdsa_gg20_keygen_batch.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_size_t, ctypes.c_int,
                                                 ctypes.POINTER(_KeygenIn), ctypes.POINTER(_KeygenOut)]
        lib._gg20_keygen_bound = True
    primes = {f: _upload(ints_to_limbs([pq[k] for pq in src], 32), mem, dev)
              for f, src, k in (("paillier_p", paillier_primes, 0), ("paillier_q", paillier_primes, 1), ("n_tilde_p", n_tilde_primes, 0),
                                ("n_tilde_q", n_tilde_primes, 1))}
    out = {"x_i": _buffer((E, 8), np.uint32, mem, dev), "vss": _buffer((E, t + 1, 16), np.uint32, mem, dev), "n": _buffer((E, 64), np.uint32, mem, dev),
           "dlog_st": _buffer((E, 3, 64), np.uint32, mem, dev), "y": _buffer((groups, 16), np.uint32, mem, dev),
           "pk": _buffer((groups, n, 16), np.uint32, mem, dev), "status": _buffer((E,), np.uint8, mem, dev),
           "bad_actors": _buffer((E,), np.uint64, mem, dev), "complete": _buffer((groups,), np.uint8, mem, dev)}
    args_in = _KeygenIn(*[_ptr(primes[f]) for f in ("paillier_p", "paillier_q", "n_tilde_p", "n_tilde_q")], *[_ptr(rnd[f]) for f in RECORD])
    args_out = _KeygenOut(*[_ptr(out[f]) for f, _ in _KeygenOut._fields_])
    eng._ck(lib.tecdsa_gg20_keygen_batch(eng._ctx, t, n, groups, mem, ctypes.byref(args_in), ctypes.byref(args_out)), "gg20_keygen")
    if mem != HOST:
        eng.sync()
    status, bad, complete = _host(out["status"]), _host(out["bad_actors"]), _host(out["complete"])
    keys = None
    if mem == HOST:
        keys = [None] * E
        nv, st, pk, y = limbs_to_ints(out["n"]), limbs_to_ints(out["dlog_st"].reshape(E * 3, 64)), limbs_to_ints(out["pk"].reshape(E, 16)), limbs_to_ints(out["y"])
        x, vss = limbs_to_ints(out["x_i"]), limbs_to_ints(out["vss"].reshape(E * (t + 1), 16))
        for g in np.flatnonzero(complete):
            rows = range(g * n, g * n + n)
            ek = [EncryptionKey(nv[r]) for r in rows]
            sts = [DLogStatement(*st[3 * r:3 * r + 3]) for r in rows]
            pks = [unpack_point(pk[r]) for r in rows]
            for i, r in enumerate(rows):
                keys[r] = LoadedLocalKey(i=i + 1, t=t, n=n, x_i=x[r], dk=DecryptionKey(*paillier_primes[r]), pk_vec=pks, paillier_key_vec=ek, h1_h2_n_tilde_vec=sts,
                                         y_sum_s=unpack_point(y[g]), vss_commitments=[unpack_point(v) for v in vss[r * (t + 1):(r + 1) * (t + 1)]])
    return KeygenResult(status, bad, complete, keys, out)
