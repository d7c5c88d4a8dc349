"""Host-side mirror of the reference's GG20 offline-stage entry (`OfflineStage::new(i, s_l, local_key)`
+ the rounds of /root/reference/src/protocols/multi_party_ecdsa/gg_2020/state_machine/sign.rs),
batched: packs `LocalKey` material and per-unit randomness into the ABI's limb records and
calls tecdsa_gg20_offline_batch.  No arithmetic happens here."""
from __future__ import annotations

import ctypes
import os
from typing import List, Optional, Sequence

import numpy as np

from . import HOST, Engine, EngineError, ints_to_limbs, limbs_to_ints, seed_words, _ptr

RND_LIMBS = 1408
# (offset, limbs) of every field of the randomness record — include/tecdsa_b200.h TECDSA_RND_*
RND = {
    "gamma_i": (0, 8), "k_i": (8, 8), "blind": (16, 8), "r_k": (24, 64),
    "beta_tag_gamma": (832, 64), "r_gamma": (896, 64), "nonce_gamma_b": (960, 8), "nonce_gamma_beta": (968, 8),
    "beta_tag_w": (976, 64), "r_w": (1040, 64), "nonce_w_b": (1104, 8), "nonce_w_beta": (1112, 8),
    "l": (1120, 8), "ped_s1": (1128, 8), "ped_s2": (1136, 8),
    "heg_s1": (1392, 8), "heg_s2": (1400, 8),
}
RND_ALICE, RND_ALICE_STRIDE = 88, 248
RND_ALICE_PARTS = ((0, 24), (24, 64), (88, 88), (176, 72))          # alpha, beta, gamma, rho
RND_PDL_PARTS = ((1144, 24), (1168, 64), (1232, 72), (1304, 88))    # alpha, beta, rho, gamma


class _Keys(ctypes.Structure):
    _fields_ = [("n_keysets", ctypes.c_size_t)] + [(n, ctypes.c_void_p) for n in
                                                   ("paillier_p", "paillier_q", "n_tilde", "h1", "h2", "x_i", "pk", "y")]


def _bind(lib):
    if getattr(lib, "_gg20_bound", False):
        return
    lib.tecdsa_keys_upload.argtypes = [ctypes.c_void_p, ctypes.POINTER(_Keys), ctypes.POINTER(ctypes.c_void_p)]
    lib.tecdsa_keys_upload_parties.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.POINTER(_Keys), ctypes.POINTER(ctypes.c_void_p)]
    lib.tecdsa_keys_free.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
    lib.tecdsa_keys_table.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p]
    lib.tecdsa_gg20_offline_batch.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t] + [ctypes.c_void_p] * 6 + [ctypes.c_int]
    lib.tecdsa_gg20_debug_field.argtypes = [ctypes.c_void_p, ctypes.c_char_p, ctypes.c_void_p, ctypes.POINTER(ctypes.c_size_t)]
    lib._gg20_bound = True


def pack_point(p) -> List[int]:
    """affine point -> x||y as one 512-bit little-endian integer (identity = 0)"""
    return 0 if p is None else p[0] | (p[1] << 256)


def unpack_point(v: int):
    return None if v == 0 else (v & ((1 << 256) - 1), v >> 256)


class KeySets:
    """Device-resident LocalKey material of several key sets of one size n (2..64 parties; key row = keyset * n + party).
    `keysets[k]` is a list of n objects with the fields of the reference's LocalKey (i, x_i, dk.p, dk.q, pk_vec,
    h1_h2_n_tilde_vec, y_sum_s) — e.g. oracle.LocalKey or any duck-typed equivalent.  Three-party key sets go through
    tecdsa_keys_upload (what the t = 1, two-signer calls take), other sizes through tecdsa_keys_upload_parties.  Every key row
    carries about 48 MB of device tables."""

    def __init__(self, eng: Engine, keysets: Sequence[Sequence]):
        _bind(eng.lib)
        sizes = {len(ks) for ks in keysets}
        if len(sizes) > 1:
            raise ValueError(f"KeySets: key sets of one size only, got sizes {sorted(sizes)}")
        self.parties = sizes.pop() if sizes else 3
        if not 2 <= self.parties <= 64:
            raise ValueError(f"KeySets: a key set has 2..64 parties, got {self.parties}")
        self.eng = eng
        self.n = len(keysets)
        rows = [lk for ks in keysets for lk in ks]
        self._bufs = dict(
            paillier_p=ints_to_limbs([lk.dk.p for lk in rows], 32), paillier_q=ints_to_limbs([lk.dk.q for lk in rows], 32),
            n_tilde=ints_to_limbs([lk.h1_h2_n_tilde_vec[lk.i - 1].N for lk in rows], 64),
            h1=ints_to_limbs([lk.h1_h2_n_tilde_vec[lk.i - 1].g for lk in rows], 64),
            h2=ints_to_limbs([lk.h1_h2_n_tilde_vec[lk.i - 1].ni for lk in rows], 64),
            x_i=ints_to_limbs([lk.x_i for lk in rows], 8),
            pk=ints_to_limbs([pack_point(lk.pk_vec[lk.i - 1]) for lk in rows], 16),
            y=ints_to_limbs([pack_point(ks[0].y_sum_s) for ks in keysets], 16))
        k = _Keys(self.n, *[self._bufs[n].ctypes.data for n in ("paillier_p", "paillier_q", "n_tilde", "h1", "h2", "x_i", "pk", "y")])
        self.handle = ctypes.c_void_p()
        if self.parties == 3:
            eng._ck(eng.lib.tecdsa_keys_upload(eng._ctx, ctypes.byref(k), ctypes.byref(self.handle)), "keys_upload")
        else:
            eng._ck(eng.lib.tecdsa_keys_upload_parties(eng._ctx, self.parties, ctypes.byref(k), ctypes.byref(self.handle)), "keys_upload_parties")

    def table(self, index: int, limbs: int) -> List[int]:
        out = np.zeros((self.n * self.parties, limbs), dtype=np.uint32)
        self.eng._ck(self.eng.lib.tecdsa_keys_table(self.eng._ctx, self.handle, index, out.ctypes.data), "keys_table")
        return limbs_to_ints(out)

    def free(self):
        if self.handle:
            self.eng.lib.tecdsa_keys_free(self.eng._ctx, self.handle)
            self.handle = ctypes.c_void_p()


def pack_randomness(units: Sequence) -> np.ndarray:
    """oracle.UnitRandomness-shaped objects -> [units][RND_LIMBS] uint32"""
    out = np.zeros((len(units), RND_LIMBS), dtype=np.uint32)

    def put(row, off, limbs, val):
        out[row, off:off + limbs] = np.frombuffer(int(val).to_bytes(4 * limbs, "little"), dtype="<u4")

    for u, r in enumerate(units):
        for name, (off, limbs) in RND.items():
            put(u, off, limbs, getattr(r, name))
        for x in range(3):
            for (o, l), v in zip(RND_ALICE_PARTS, r.alice[x]):
                put(u, RND_ALICE + x * RND_ALICE_STRIDE + o, l, v)
        for (o, l), v in zip(RND_PDL_PARTS, r.pdl):
            put(u, o, l, v)
    return out


class OfflineResult:
    def __init__(self, status, R, sigma, t_vec, digest):
        self.status, self.R, self.sigma, self.t_vec, self.digest = status, R, sigma, t_vec, digest


def offline_batch(eng: Engine, keys: KeySets, sessions: Sequence[Sequence[int]], rnd: np.ndarray, mem: int = HOST) -> OfflineResult:
    """sessions[s] = (keyset, party0, party1) with parties 0-based; rnd from pack_randomness()."""
    _bind(eng.lib)
    n = len(sessions)
    sess = np.ascontiguousarray(np.array(sessions, dtype=np.uint32).reshape(n, 3))
    U = 2 * n
    assert rnd.shape == (U, RND_LIMBS)
    status = np.full(U, 255, dtype=np.uint8)
    R = np.zeros((U, 16), np.uint32); sigma = np.zeros((U, 8), np.uint32)
    tvec = np.zeros((U, 32), np.uint32); digest = np.zeros((U, 8), np.uint32)
    eng._ck(eng.lib.tecdsa_gg20_offline_batch(eng._ctx, keys.handle, _ptr(sess), n, _ptr(rnd), _ptr(status), _ptr(R), _ptr(sigma),
                                              _ptr(tvec), _ptr(digest), mem), "gg20_offline_batch")
    return OfflineResult(status, R, sigma, tvec, digest)


def offline_raw(eng: Engine, keys: KeySets, sessions, n_sessions: int, rnd, status, R, sigma, t_vec, digest, mem: int = HOST):
    """tecdsa_gg20_offline_batch on caller buffers (numpy for HOST, torch CUDA tensors for DEVICE)"""
    _bind(eng.lib)
    eng._ck(eng.lib.tecdsa_gg20_offline_batch(eng._ctx, keys.handle, _ptr(sessions), n_sessions, _ptr(rnd), _ptr(status), _ptr(R), _ptr(sigma),
                                              _ptr(t_vec), _ptr(digest), mem), "gg20_offline_batch")


def sign_batch(eng: Engine, keys: KeySets, sessions: np.ndarray, message: np.ndarray, R: np.ndarray, sigma: np.ndarray, k: np.ndarray):
    """The online step for a batch of completed sessions (`phase7_local_sig`, `output_signature`, `verify`; party_i.rs:850-936):
    message [n][8], R [2n][16], sigma [2n][8], k [2n][8] (uint32 limbs) -> dict(s_i [2n][8], r [n][8], s [n][8], recid [n], status [n])"""
    _bind(eng.lib)
    lib = eng.lib
    if not getattr(lib, "_sign_bound", False):
        lib.tecdsa_gg20_sign_batch.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t] + [ctypes.c_void_p] * 9 + [ctypes.c_int]
        lib._sign_bound = True
    sessions = np.ascontiguousarray(sessions, dtype=np.uint32).reshape(-1, 3)
    n = sessions.shape[0]
    ins = [np.ascontiguousarray(x, dtype=np.uint32) for x in (message, R, sigma, k)]
    s_i, r, s = np.zeros((2 * n, 8), np.uint32), np.zeros((n, 8), np.uint32), np.zeros((n, 8), np.uint32)
    recid, status = np.zeros(n, np.uint8), np.full(n, 255, np.uint8)
    eng._ck(lib.tecdsa_gg20_sign_batch(eng._ctx, keys.handle, _ptr(sessions), n, *[_ptr(x) for x in ins], _ptr(s_i), _ptr(r), _ptr(s), _ptr(recid), _ptr(status), HOST),
            "gg20_sign_batch")
    return {"s_i": s_i, "r": r, "s": s, "recid": recid, "status": status}


# TECDSA_RNDS_*: the sampler's stream id of every field of the randomness record (Alice fields: RNDS_ALICE + 4 * statement + part)
RNDS = {"gamma": 0, "k": 1, "blind": 2, "r_k": 3, "beta_tag_gamma": 16, "r_gamma": 17, "nonce_gamma_b": 18, "nonce_gamma_beta": 19,
        "beta_tag_w": 20, "r_w": 21, "nonce_w_b": 22, "nonce_w_beta": 23, "l": 24, "ped_s1": 25, "ped_s2": 26,
        "pdl_alpha": 27, "pdl_beta": 28, "pdl_rho": 29, "pdl_gamma": 30, "heg_s1": 31, "heg_s2": 32}
RNDS_ALICE = 4


def fresh_seed(seed: Optional[bytes] = None) -> bytes:
    """The caller's 32-byte seed, or a fresh one from the OS CSPRNG — the one place the product touches it.  A seed drawn here is
    used for the one call it was drawn for and is never returned to the caller, stored or logged."""
    return os.urandom(32) if seed is None else bytes(seed)


def sample_randomness(eng: Engine, keys: KeySets, sessions, seed: Optional[bytes] = None, first_unit: int = 0, mem: int = HOST, rnd=None, status=None):
    """The sampling half of the reference's `MessageA::a`, `MessageB::b`, `AliceProof::generate`, `PDLwSlackProof::prove`,
    `SignKeys::create` for a batch of sessions (tecdsa_gg20_sample_randomness): -> (rnd [2n][RND_LIMBS], status [2n]), the record
    `offline_batch` takes, every field a function of (seed, first_unit + unit, field, key material).  seed=None draws a fresh one.
    A (seed, unit id) pair must never be used twice: fresh seed per call, or one seed with disjoint first_unit ranges.
    mem=DEVICE: sessions, rnd and status are the caller's CUDA tensors and the record never reaches the host."""
    _bind(eng.lib)
    lib = eng.lib
    if not getattr(lib, "_gg20_sample_bound", False):
        V = ctypes.c_void_p
        lib.tecdsa_gg20_sample_randomness.argtypes = [V, V, V, ctypes.c_size_t, V, ctypes.c_uint64, V, V, ctypes.c_int]
        lib._gg20_sample_bound = True
    if mem == HOST:
        sessions = np.ascontiguousarray(np.asarray(sessions, dtype=np.uint32).reshape(-1, 3))
        n = sessions.shape[0]
        rnd = np.zeros((2 * n, RND_LIMBS), dtype=np.uint32)
        status = np.full(2 * n, 255, dtype=np.uint8)
    else:
        n = sessions.shape[0]
    sw = seed_words(fresh_seed(seed))
    try:
        eng._ck(lib.tecdsa_gg20_sample_randomness(eng._ctx, keys.handle, _ptr(sessions), n, _ptr(sw), first_unit, _ptr(rnd), _ptr(status), mem),
                "gg20_sample_randomness")
    finally:
        sw[:] = 0
    return rnd, status


def debug_field(eng: Engine, name: str, units: int) -> np.ndarray:
    _bind(eng.lib)
    n = ctypes.c_size_t()
    eng._ck(eng.lib.tecdsa_gg20_debug_field(eng._ctx, name.encode(), None, ctypes.byref(n)), "debug_field")
    out = np.zeros((units, n.value), dtype=np.uint32)
    eng._ck(eng.lib.tecdsa_gg20_debug_field(eng._ctx, name.encode(), out.ctypes.data, ctypes.byref(n)), "debug_field")
    return out


# ----------------------------------------------------------------------------- synthetic batches (bench / scale tests)
_Q = 0xFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFEBAAEDCE6AF48A03BBFD25E8CD0364141


def synthetic_batch(keysets: Sequence[Sequence], n_sessions: int, seed: int):
    """Random valid inputs for `n_sessions` two-signer sessions over the given key sets: returns
    (sessions [n,3] uint32, rnd [2n, RND_LIMBS] uint32).  Every value is drawn uniformly with one
    bit less than its reference bound (so it is always in range; the bounds are those of
    `sample_unit` in oracle/sampling.py), vectorised with numpy so that 10^5 units take seconds."""
    rng = np.random.default_rng(seed)
    pairs = [(0, 1), (0, 2), (1, 2), (1, 0), (2, 0), (2, 1)]
    n_ks = len(keysets)
    ks_idx = rng.integers(0, n_ks, size=n_sessions)
    pr_idx = rng.integers(0, len(pairs), size=n_sessions)
    sessions = np.zeros((n_sessions, 3), dtype=np.uint32)
    sessions[:, 0] = ks_idx
    sessions[:, 1] = [pairs[i][0] for i in pr_idx]
    sessions[:, 2] = [pairs[i][1] for i in pr_idx]
    U = 2 * n_sessions
    rnd = np.zeros((U, RND_LIMBS), dtype=np.uint32)

    def fill(rows, off, limbs, bits):
        """uniform `bits`-bit values (lowest limb forced odd/non-zero where it matters is not needed)"""
        full, rem = divmod(bits, 32)
        block = rng.integers(0, 2 ** 32, size=(len(rows), limbs), dtype=np.uint32)
        block[:, full + (1 if rem else 0):] = 0
        if rem:
            block[:, full] &= np.uint32((1 << rem) - 1)
        block[:, 0] |= 1                      # never zero
        rnd[np.asarray(rows)[:, None], off + np.arange(limbs)[None, :]] = block

    all_rows = np.arange(U)
    for name in ("gamma_i", "k_i", "nonce_gamma_b", "nonce_gamma_beta", "nonce_w_b", "nonce_w_beta", "l", "ped_s1", "ped_s2", "heg_s1", "heg_s2"):
        fill(all_rows, RND[name][0], 8, 255)
    fill(all_rows, RND["blind"][0], 8, 256)
    q3_bits = (_Q ** 3).bit_length() - 1
    # the remaining fields depend on the moduli of the unit's own / peer's key rows
    unit_ks = np.repeat(ks_idx, 2)
    own = np.stack([sessions[:, 1], sessions[:, 2]], axis=1).reshape(-1)
    peer = np.stack([sessions[:, 2], sessions[:, 1]], axis=1).reshape(-1)
    for k in range(n_ks):
        for party in range(3):
            lk = keysets[k][party]
            n_bits = (lk.dk.p * lk.dk.q).bit_length() - 1
            rows = all_rows[(unit_ks == k) & (own == party)]
            if len(rows):
                fill(rows, RND["r_k"][0], 64, n_bits)
                fill(rows, RND_PDL_PARTS[1][0], 64, n_bits)                       # pdl beta
                for x in range(3):
                    nt = keysets[k][x].h1_h2_n_tilde_vec[x].N
                    base = RND_ALICE + x * RND_ALICE_STRIDE
                    fill(rows, base + RND_ALICE_PARTS[0][0], 24, q3_bits)
                    fill(rows, base + RND_ALICE_PARTS[1][0], 64, n_bits)
                    fill(rows, base + RND_ALICE_PARTS[2][0], 88, (_Q ** 3 * nt).bit_length() - 1)
                    fill(rows, base + RND_ALICE_PARTS[3][0], 72, (_Q * nt).bit_length() - 1)
            rows = all_rows[(unit_ks == k) & (peer == party)]
            if len(rows):
                for name in ("beta_tag_gamma", "r_gamma", "beta_tag_w", "r_w"):
                    fill(rows, RND[name][0], 64, n_bits)
                nt = lk.h1_h2_n_tilde_vec[party].N                                # PDL is proved against the peer's statement
                fill(rows, RND_PDL_PARTS[0][0], 24, q3_bits)
                fill(rows, RND_PDL_PARTS[2][0], 72, (_Q * nt).bit_length() - 1)
                fill(rows, RND_PDL_PARTS[3][0], 88, (_Q ** 3 * nt).bit_length() - 1)
    return sessions, rnd


# ----------------------------------------------------------------------------- L2: AliceProof (MtA range proof) batched
def _bind_l2(lib):
    if getattr(lib, "_l2_bound", False):
        return
    V, S, I = ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int
    lib.tecdsa_alice_proof_generate_batch.argtypes = [V] * 16 + [S, I]
    lib.tecdsa_alice_proof_verify_batch.argtypes = [V] * 11 + [S, I]
    lib._l2_bound = True


def alice_proof_generate(eng: Engine, keys: KeySets, ek_row, st_row, a, cipher, r, alpha, beta, gamma, rho):
    """Batched `AliceProof::generate` (range_proofs.rs:160-193) with explicit randomness; returns dict of int lists."""
    _bind_l2(eng.lib)
    n = len(a)
    er, sr = np.asarray(ek_row, dtype=np.uint32), np.asarray(st_row, dtype=np.uint32)
    ins = [ints_to_limbs(a, 8), ints_to_limbs(cipher, 128), ints_to_limbs(r, 64), ints_to_limbs(alpha, 24), ints_to_limbs(beta, 64),
           ints_to_limbs(gamma, 88), ints_to_limbs(rho, 72)]
    outs = {k: np.zeros((n, l), dtype=np.uint32) for k, l in (("z", 64), ("e", 8), ("s", 64), ("s1", 28), ("s2", 92))}
    eng._ck(eng.lib.tecdsa_alice_proof_generate_batch(eng._ctx, keys.handle, _ptr(er), _ptr(sr), *[_ptr(x) for x in ins],
                                                      *[_ptr(outs[k]) for k in ("z", "e", "s", "s1", "s2")], n, HOST), "alice_proof_generate")
    return {k: limbs_to_ints(v) for k, v in outs.items()}


class _Screen:
    """Untrusted proof fields arrive as arbitrary integers; the ABI slots have fixed widths.  A field that is negative or wider
    than its slot can never verify (the reference compares / hashes the full value: `s1 > q^3`, range_proofs.rs:118, or a
    challenge mismatch), so it is replaced by 0 and that ONE proof is marked rejected after the call — it must not abort the
    whole batch with an OverflowError in the limb packing."""

    def __init__(self, n: int):
        self.bad = np.zeros(n, dtype=bool)
        self.range_bad = np.zeros(n, dtype=bool)

    def limbs(self, vals, k: int, is_range_field: bool = False) -> np.ndarray:
        out = []
        for i, v in enumerate(vals):
            v = int(v)
            if v < 0 or v >> (32 * k):
                (self.range_bad if is_range_field and v > 0 else self.bad)[i] = True
                v = 0
            out.append(v)
        return ints_to_limbs(out, k)

    def apply(self, status: np.ndarray, code: int, range_code: int = None) -> np.ndarray:
        status[self.bad] = code
        status[self.range_bad] = code if range_code is None else range_code
        return status


def alice_proof_verify(eng: Engine, keys: KeySets, ek_row, st_row, cipher, z, e, s, s1, s2) -> np.ndarray:
    """Batched `AliceProof::verify` (range_proofs.rs:105-156): status byte per proof (0 = accept)."""
    _bind_l2(eng.lib)
    n = len(z)
    er, sr = np.asarray(ek_row, dtype=np.uint32), np.asarray(st_row, dtype=np.uint32)
    sc = _Screen(n)
    ins = [sc.limbs(cipher, 128), sc.limbs(z, 64), sc.limbs(e, 8), sc.limbs(s, 64), sc.limbs(s1, 28, True), sc.limbs(s2, 92)]
    status = np.full(n, 255, dtype=np.uint8)
    eng._ck(eng.lib.tecdsa_alice_proof_verify_batch(eng._ctx, keys.handle, _ptr(er), _ptr(sr), *[_ptr(x) for x in ins], _ptr(status), n, HOST),
            "alice_proof_verify")
    return sc.apply(status, 5, 3)            # TECDSA_ST_HASH_MISMATCH; an over-wide s1 is the `s1 > q^3` reject (TECDSA_ST_RANGE)


# ----------------------------------------------------------------------------- L2: PDLwSlack and Bob proofs, batched
def _bind_l2b(lib):
    if getattr(lib, "_l2b_bound", False):
        return
    V, S, I = ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int
    lib.tecdsa_pdl_prove_batch.argtypes = [V] * 20 + [S, I]
    lib.tecdsa_pdl_verify_batch.argtypes = [V] * 15 + [S, I]
    lib.tecdsa_bob_proof_generate_batch.argtypes = [V, V, V, V, I] + [V] * 21 + [S, I]
    lib.tecdsa_bob_proof_verify_batch.argtypes = [V] * 17 + [S, I]
    lib._l2b_bound = True


def _rows(x):
    return np.asarray(x, dtype=np.uint32)


def _pts(ps):
    return ints_to_limbs([pack_point(p) for p in ps], 16)


def pdl_prove(eng, keys, ek_row, st_row, x, r, cipher, Q, G, alpha, beta, rho, gamma):
    """Batched `PDLwSlackProof::prove` (zk_pdl_with_slack/mod.rs:68-125) with explicit randomness."""
    _bind_l2b(eng.lib)
    n = len(x)
    ins = [_rows(ek_row), _rows(st_row), ints_to_limbs(x, 8), ints_to_limbs(r, 64), ints_to_limbs(cipher, 128), _pts(Q), _pts(G),
           ints_to_limbs(alpha, 24), ints_to_limbs(beta, 64), ints_to_limbs(rho, 72), ints_to_limbs(gamma, 88)]
    outs = {k: np.zeros((n, l), dtype=np.uint32) for k, l in (("z", 64), ("u1", 16), ("u2", 128), ("u3", 64), ("s1", 28), ("s2", 64), ("s3", 92))}
    eng._ck(eng.lib.tecdsa_pdl_prove_batch(eng._ctx, keys.handle, *[_ptr(a) for a in ins], *[_ptr(outs[k]) for k in ("z", "u1", "u2", "u3", "s1", "s2", "s3")],
                                           n, HOST), "pdl_prove")
    res = {k: limbs_to_ints(v) for k, v in outs.items()}
    res["u1"] = [unpack_point(v) for v in res["u1"]]
    return res


def pdl_verify(eng, keys, ek_row, st_row, cipher, Q, G, z, u1, u2, u3, s1, s2, s3) -> np.ndarray:
    _bind_l2b(eng.lib)
    n = len(z)
    sc = _Screen(n)
    ins = [_rows(ek_row), _rows(st_row), sc.limbs(cipher, 128), _pts(Q), _pts(G), sc.limbs(z, 64), _pts(u1), sc.limbs(u2, 128),
           sc.limbs(u3, 64), sc.limbs(s1, 28), sc.limbs(s2, 64), sc.limbs(s3, 92)]
    status = np.full(n, 255, dtype=np.uint8)
    eng._ck(eng.lib.tecdsa_pdl_verify_batch(eng._ctx, keys.handle, *[_ptr(a) for a in ins], _ptr(status), n, HOST), "pdl_verify")
    return sc.apply(status, 6)               # TECDSA_ST_PDL_VERIFY


def bob_proof_generate(eng, keys, ek_row, st_row, check, a_enc, mta_enc, b, beta_prim, r, alpha, beta, gamma, ro, ro_prim, sigma, tau):
    """Batched `BobProof::generate` (range_proofs.rs:414-487); check=True is the MtAwc variant (returns u too)."""
    _bind_l2b(eng.lib)
    n = len(b)
    ins = [ints_to_limbs(a_enc, 128), ints_to_limbs(mta_enc, 128), ints_to_limbs(b, 8), ints_to_limbs(beta_prim, 64), ints_to_limbs(r, 64),
           ints_to_limbs(alpha, 24), ints_to_limbs(beta, 64), ints_to_limbs(gamma, 80), ints_to_limbs(ro, 72), ints_to_limbs(ro_prim, 88),
           ints_to_limbs(sigma, 72), ints_to_limbs(tau, 88)]
    names = (("t", 64), ("z", 64), ("e", 8), ("s", 64), ("s1", 28), ("s2", 92), ("t1", 84), ("t2", 92), ("u", 16))
    outs = {k: np.zeros((n, l), dtype=np.uint32) for k, l in names}
    er, sr = _rows(ek_row), _rows(st_row)
    eng._ck(eng.lib.tecdsa_bob_proof_generate_batch(eng._ctx, keys.handle, _ptr(er), _ptr(sr), 1 if check else 0, *[_ptr(a) for a in ins],
                                                    *[_ptr(outs[k]) for k, _ in names], n, HOST), "bob_proof_generate")
    res = {k: limbs_to_ints(v) for k, v in outs.items()}
    res["u"] = [unpack_point(v) for v in res["u"]] if check else None
    return res


def bob_proof_verify(eng, keys, ek_row, st_row, a_enc, mta_out, pf, X=None, u=None) -> np.ndarray:
    """Batched `BobProof::verify` (X is None) / `BobProofExt::verify` (X = G*b, u from the proof)."""
    _bind_l2b(eng.lib)
    n = len(pf["z"])
    sc = _Screen(n)
    ins = [_rows(ek_row), _rows(st_row), sc.limbs(a_enc, 128), sc.limbs(mta_out, 128), sc.limbs(pf["t"], 64), sc.limbs(pf["z"], 64),
           sc.limbs(pf["e"], 8), sc.limbs(pf["s"], 64), sc.limbs(pf["s1"], 28, True), sc.limbs(pf["s2"], 92), sc.limbs(pf["t1"], 84),
           sc.limbs(pf["t2"], 92)]
    Xa = _pts(X) if X is not None else None
    Ua = _pts(u) if u is not None else None
    status = np.full(n, 255, dtype=np.uint8)
    eng._ck(eng.lib.tecdsa_bob_proof_verify_batch(eng._ctx, keys.handle, *[_ptr(a) for a in ins], _ptr(Xa), _ptr(Ua), _ptr(status), n, HOST), "bob_proof_verify")
    return sc.apply(status, 5, 3)


# ----------------------------------------------------------------------------- curv sigma proofs / hashes, batched
def _bind_sigma(lib):
    if getattr(lib, "_sigma_bound", False):
        return
    V, S, I = ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int
    lib.tecdsa_dlog_prove_batch.argtypes = [V, V, V, V, S, I]
    lib.tecdsa_dlog_verify_batch.argtypes = [V, V, V, S, I]
    lib.tecdsa_pedersen_prove_batch.argtypes = [V] * 7 + [S, I]
    lib.tecdsa_pedersen_verify_batch.argtypes = [V, V, V, V, S, I]
    lib.tecdsa_heg_prove_batch.argtypes = [V] * 9 + [S, I]
    lib.tecdsa_heg_verify_batch.argtypes = [V] * 6 + [S, I]
    lib.tecdsa_sha256_bigints_batch.argtypes = [V, V, V, I, V, S, I]
    lib.tecdsa_hash_commitment_batch.argtypes = [V, V, V, V, S, I]
    lib._sigma_bound = True


def dlog_prove(eng, sk, nonce):
    """Batched curv `DLogProof::prove`; returns (n, 40) uint32: pk 16 | T 16 | response 8."""
    _bind_sigma(eng.lib)
    a, b = ints_to_limbs(sk, 8), ints_to_limbs(nonce, 8)
    out = np.zeros((len(sk), 40), dtype=np.uint32)
    eng._ck(eng.lib.tecdsa_dlog_prove_batch(eng._ctx, _ptr(a), _ptr(b), _ptr(out), len(sk), HOST), "dlog_prove")
    return out


def dlog_verify(eng, proofs: np.ndarray) -> np.ndarray:
    _bind_sigma(eng.lib)
    st = np.full(proofs.shape[0], 255, dtype=np.uint8)
    p = np.ascontiguousarray(proofs, dtype=np.uint32)
    eng._ck(eng.lib.tecdsa_dlog_verify_batch(eng._ctx, _ptr(p), _ptr(st), p.shape[0], HOST), "dlog_verify")
    return st


def pedersen_prove(eng, m, r, s1, s2):
    _bind_sigma(eng.lib)
    ins = [ints_to_limbs(x, 8) for x in (m, r, s1, s2)]
    com, pf = np.zeros((len(m), 16), np.uint32), np.zeros((len(m), 64), np.uint32)
    eng._ck(eng.lib.tecdsa_pedersen_prove_batch(eng._ctx, *[_ptr(a) for a in ins], _ptr(com), _ptr(pf), len(m), HOST), "pedersen_prove")
    return com, pf


def pedersen_verify(eng, com, pf) -> np.ndarray:
    _bind_sigma(eng.lib)
    st = np.full(com.shape[0], 255, dtype=np.uint8)
    eng._ck(eng.lib.tecdsa_pedersen_verify_batch(eng._ctx, _ptr(com), _ptr(pf), _ptr(st), com.shape[0], HOST), "pedersen_verify")
    return st


def heg_prove(eng, G, D, E, x, r, s1, s2):
    _bind_sigma(eng.lib)
    ins = [_pts(G), _pts(D), _pts(E)] + [ints_to_limbs(v, 8) for v in (x, r, s1, s2)]
    pf = np.zeros((len(x), 48), np.uint32)
    eng._ck(eng.lib.tecdsa_heg_prove_batch(eng._ctx, *[_ptr(a) for a in ins], _ptr(pf), len(x), HOST), "heg_prove")
    return pf


def heg_verify(eng, G, D, E, pf) -> np.ndarray:
    _bind_sigma(eng.lib)
    st = np.full(pf.shape[0], 255, dtype=np.uint8)
    ins = [_pts(G), _pts(D), _pts(E)]
    eng._ck(eng.lib.tecdsa_heg_verify_batch(eng._ctx, *[_ptr(a) for a in ins], _ptr(pf), _ptr(st), pf.shape[0], HOST), "heg_verify")
    return st


def sha256_bigints(eng, rows, item_limbs):
    """rows: list of tuples of ints (one tuple per digest), item_limbs: limbs reserved per item."""
    _bind_sigma(eng.lib)
    n = len(rows)
    data = np.concatenate([ints_to_limbs([row[j] for row in rows], l) for j, l in enumerate(item_limbs)], axis=1)
    data = np.ascontiguousarray(data)
    il = (ctypes.c_int * len(item_limbs))(*item_limbs)
    out = np.zeros((n, 8), dtype=np.uint32)
    eng._ck(eng.lib.tecdsa_sha256_bigints_batch(eng._ctx, _ptr(data), il, len(item_limbs), _ptr(out), n, HOST), "sha256_bigints")
    return limbs_to_ints(out)


def hash_commitment(eng, points, blinds):
    _bind_sigma(eng.lib)
    P, B = _pts(points), ints_to_limbs(blinds, 8)
    out = np.zeros((len(blinds), 8), dtype=np.uint32)
    eng._ck(eng.lib.tecdsa_hash_commitment_batch(eng._ctx, _ptr(P), _ptr(B), _ptr(out), len(blinds), HOST), "hash_commitment")
    return limbs_to_ints(out)


# ----------------------------------------------------------------------------- L2: MtA messages, batched
def _bind_mta(lib):
    if getattr(lib, "_mta_bound", False):
        return
    V, S, I = ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int
    lib.tecdsa_mta_message_a_batch.argtypes = [V, V, V, V, I] + [V] * 12 + [S, I]
    lib.tecdsa_mta_message_b_batch.argtypes = [V, V, V, V, I] + [V] * 16 + [S, I]
    lib.tecdsa_mta_get_alpha_batch.argtypes = [V] * 10 + [S, I]
    lib._mta_bound = True


def mta_message_a(eng, keys, ek_row, st_rows, a, r, proof_rand):
    """Batched `MessageA::a_with_predefined_randomness`.  st_rows: [n][n_st] key rows; proof_rand[i][x] =
    (alpha, beta, gamma, rho).  Returns (c list, dict of [n][n_st] int lists)."""
    _bind_mta(eng.lib)
    n = len(a)
    n_st = len(st_rows[0]) if n else 0
    flat = [pr for inst in proof_rand for pr in inst]
    ins = [ints_to_limbs(a, 8), ints_to_limbs(r, 64)] + [ints_to_limbs([p[j] for p in flat], l) for j, l in enumerate((24, 64, 88, 72))]
    c = np.zeros((n, 128), np.uint32)
    outs = {k: np.zeros((n * n_st, l), np.uint32) for k, l in (("z", 64), ("e", 8), ("s", 64), ("s1", 28), ("s2", 92))}
    er, sr = _rows(ek_row), np.ascontiguousarray(np.asarray(st_rows, dtype=np.uint32).reshape(-1))
    eng._ck(eng.lib.tecdsa_mta_message_a_batch(eng._ctx, keys.handle, _ptr(er), _ptr(sr), n_st, *[_ptr(x) for x in ins], _ptr(c),
                                               *[_ptr(outs[k]) for k in ("z", "e", "s", "s1", "s2")], n, HOST), "mta_message_a")
    proofs = {k: [limbs_to_ints(v)[i * n_st:(i + 1) * n_st] for i in range(n)] for k, v in outs.items()}
    return limbs_to_ints(c), proofs


def mta_message_b(eng, keys, ek_row, st_rows, b, c_a, proofs, randomness, beta_tag, nonce_b, nonce_beta):
    """Batched `MessageB::b_with_predefined_randomness`; proofs as returned by mta_message_a."""
    _bind_mta(eng.lib)
    n = len(b)
    n_st = len(st_rows[0]) if n else 0
    flat = {k: [v for inst in proofs[k] for v in inst] for k in ("z", "e", "s", "s1", "s2")}
    er, sr = _rows(ek_row), np.ascontiguousarray(np.asarray(st_rows, dtype=np.uint32).reshape(-1))
    # the peer's MessageA is untrusted: an over-wide field of any of its range proofs makes that MessageB Err(InvalidKey)
    scp, sca = _Screen(n * n_st), _Screen(n)
    ins = [ints_to_limbs(b, 8), sca.limbs(c_a, 128), scp.limbs(flat["z"], 64), scp.limbs(flat["e"], 8), scp.limbs(flat["s"], 64),
           scp.limbs(flat["s1"], 28), scp.limbs(flat["s2"], 92), ints_to_limbs(randomness, 64), ints_to_limbs(beta_tag, 64),
           ints_to_limbs(nonce_b, 8), ints_to_limbs(nonce_beta, 8)]
    c_b, bp, btp, beta = np.zeros((n, 128), np.uint32), np.zeros((n, 40), np.uint32), np.zeros((n, 40), np.uint32), np.zeros((n, 8), np.uint32)
    status = np.full(n, 255, np.uint8)
    eng._ck(eng.lib.tecdsa_mta_message_b_batch(eng._ctx, keys.handle, _ptr(er), _ptr(sr), n_st, *[_ptr(x) for x in ins], _ptr(c_b), _ptr(bp), _ptr(btp),
                                               _ptr(beta), _ptr(status), n, HOST), "mta_message_b")
    rejected = sca.bad | sca.range_bad
    if n_st:
        rejected |= (scp.bad | scp.range_bad).reshape(n, n_st).any(axis=1)
    status[rejected] = 2                     # TECDSA_ST_INVALID_KEY (mta/mod.rs:120,130)
    return limbs_to_ints(c_b), bp, btp, limbs_to_ints(beta), status


def mta_get_alpha(eng, keys, dk_row, a, c_b, b_proof, beta_tag_proof):
    """Batched `MessageB::verify_proofs_get_alpha` -> (alpha list, alpha' list, status)."""
    _bind_mta(eng.lib)
    n = len(a)
    ins = [_rows(dk_row), ints_to_limbs(a, 8), ints_to_limbs(c_b, 128), np.ascontiguousarray(b_proof), np.ascontiguousarray(beta_tag_proof)]
    alpha, plain = np.zeros((n, 8), np.uint32), np.zeros((n, 64), np.uint32)
    status = np.full(n, 255, np.uint8)
    eng._ck(eng.lib.tecdsa_mta_get_alpha_batch(eng._ctx, keys.handle, *[_ptr(x) for x in ins], _ptr(alpha), _ptr(plain), _ptr(status), n, HOST), "mta_get_alpha")
    return limbs_to_ints(alpha), limbs_to_ints(plain), status
