"""multi-party-ecdsa_b200 — host-side mirror of the reference's arithmetic surface over the
C-ABI library (include/tecdsa_b200.h).

The reference (ZenGo-X/multi-party-ecdsa) is Rust and its seam is the curv-kzen
`BigInt` / kzen-paillier trait surface; there is no Rust toolchain in this image, so this
module is the thin host layer the tests and the bench drive: same operation names and
argument meaning (`mod_pow(base, exponent, modulus)` = `BigInt::mod_pow`,
/root/reference/src/utilities/mta/range_proofs.rs:52), batched over the leading axis.
It only packs limbs and calls the shared library through ctypes — there is NO CPU
arithmetic fallback here: if the CUDA library is missing or no GPU is present every call
raises.  (The directory name has a hyphen; import it with `load_package()` from
__graft_entry__.py or tests/conftest.py, which registers it as `mpecdsa_b200`.)
"""
from __future__ import annotations

import ctypes
import os
from typing import Iterable, List, Optional, Sequence

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
# TECDSA_B200_LIB names another build of the same library (A/B measurements of kernel variants)
LIB_PATH = os.environ.get("TECDSA_B200_LIB") or os.path.join(_HERE, "libtecdsa_b200.so")

HOST, DEVICE = 0, 1
ST_OK, ST_EVEN_MODULUS, ST_INVALID_KEY, ST_RANGE, ST_NOT_INVERTIBLE, ST_HASH_MISMATCH = 0, 1, 2, 3, 4, 5
ST_PDL_VERIFY, ST_PHASE5_BAD_SUM, ST_PHASE6, ST_INVALID_SIG, ST_PROOF, ST_COMMITMENT, ST_INVALID_SS = 6, 7, 8, 9, 10, 11, 12
ST_SAMPLING = 13
SAMPLE_BITS, SAMPLE_BELOW, SAMPLE_UNIT, SAMPLE_RANGE1, SAMPLE_SCALAR = 0, 1, 2, 3, 4      # TECDSA_SAMPLE_*

# every symbol include/tecdsa_b200.h declares (checked by tests/test_abi.py)
EXPORTS = [
    "tecdsa_ctx_create", "tecdsa_ctx_destroy", "tecdsa_ctx_sync", "tecdsa_last_error", "tecdsa_ctx_set_tpi", "tecdsa_ctx_set_option",
    "tecdsa_ctx_last_kernel_ms", "tecdsa_ctx_launch_count", "tecdsa_modexp_batch", "tecdsa_imad_peak", "tecdsa_imad_peak_chained",
    "tecdsa_keys_upload", "tecdsa_keys_free", "tecdsa_keys_table", "tecdsa_gg20_offline_batch", "tecdsa_gg20_debug_field",
    "tecdsa_modmul_batch", "tecdsa_modinv_batch", "tecdsa_secp_mul_batch", "tecdsa_paillier_encrypt_batch", "tecdsa_paillier_mul_batch",
    "tecdsa_paillier_add_batch", "tecdsa_paillier_decrypt_batch", "tecdsa_alice_proof_generate_batch", "tecdsa_alice_proof_verify_batch",
    "tecdsa_pdl_prove_batch", "tecdsa_pdl_verify_batch", "tecdsa_bob_proof_generate_batch", "tecdsa_bob_proof_verify_batch",
    "tecdsa_dlog_prove_batch", "tecdsa_dlog_verify_batch", "tecdsa_pedersen_prove_batch", "tecdsa_pedersen_verify_batch",
    "tecdsa_heg_prove_batch", "tecdsa_heg_verify_batch", "tecdsa_sha256_bigints_batch", "tecdsa_hash_commitment_batch",
    "tecdsa_mta_message_a_batch", "tecdsa_mta_message_b_batch", "tecdsa_mta_get_alpha_batch",
    "tecdsa_correct_key_verify_batch", "tecdsa_composite_dlog_verify_batch", "tecdsa_vss_validate_share_batch",
    "tecdsa_gg20_pack_records", "tecdsa_gather_results", "tecdsa_nccl_unique_id", "tecdsa_nccl_comm_create", "tecdsa_nccl_comm_destroy",
    "tecdsa_gg20_offline_records", "tecdsa_gg20_sign_batch", "tecdsa_ctx_work", "tecdsa_ctx_profile", "tecdsa_ctx_profile_read",
    "tecdsa_secp_add_batch", "tecdsa_secp_sub_batch", "tecdsa_secp_compress_batch", "tecdsa_secp_decompress_batch", "tecdsa_secp_scalar_mul_batch",
    "tecdsa_secp_scalar_add_batch", "tecdsa_secp_scalar_sub_batch", "tecdsa_secp_scalar_inv_batch", "tecdsa_secp_scalar_from_bigint_batch",
    "tecdsa_wide_muladd_batch", "tecdsa_unit_mod_check_batch", "tecdsa_sha256_batch",
    "tecdsa_paillier_open_batch", "tecdsa_ecddh_prove_batch", "tecdsa_ecddh_verify_batch",
    "tecdsa_correct_key_prove_batch", "tecdsa_composite_dlog_prove_batch", "tecdsa_vss_share_batch", "tecdsa_h1_h2_n_tilde_batch",
    "tecdsa_l17_eph_create_batch", "tecdsa_l17_eph_verify_batch", "tecdsa_l17_partial_sig_batch", "tecdsa_l17_sign_batch", "tecdsa_l17_verify_batch",
    "tecdsa_zkpdl_verifier_message1_batch", "tecdsa_zkpdl_prover_message1_batch", "tecdsa_zkpdl_prover_message2_batch",
    "tecdsa_zkpdl_verifier_finalize_batch",
    "tecdsa_gg18_phase4_batch", "tecdsa_gg18_local_sig_batch", "tecdsa_gg18_phase5a_batch", "tecdsa_gg18_phase5c_batch", "tecdsa_gg18_phase5d_batch",
    "tecdsa_gg18_output_signature_batch",
    "tecdsa_sample_batch", "tecdsa_gg20_sample_randomness", "tecdsa_gg20_keygen_batch",
    "tecdsa_keys_upload_parties", "tecdsa_gg20_offline_general_batch", "tecdsa_gg18_signing_batch",
]


class EngineError(RuntimeError):
    pass


_lib = None


def load_library() -> ctypes.CDLL:
    """dlopen the in-tree CUDA library; fail loudly when it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise EngineError(f"{LIB_PATH} not built — run `python -c 'import __graft_entry__ as g; g.build()'`")
        lib = ctypes.CDLL(LIB_PATH)
        lib.tecdsa_last_error.restype = ctypes.c_char_p
        lib.tecdsa_ctx_launch_count.restype = ctypes.c_uint64
        lib.tecdsa_ctx_launch_count.argtypes = [ctypes.c_void_p]
        lib.tecdsa_ctx_create.argtypes = [ctypes.POINTER(ctypes.c_void_p), ctypes.c_int, ctypes.c_void_p]
        lib.tecdsa_ctx_destroy.argtypes = [ctypes.c_void_p]
        lib.tecdsa_ctx_sync.argtypes = [ctypes.c_void_p]
        lib.tecdsa_ctx_set_tpi.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int]
        lib.tecdsa_ctx_last_kernel_ms.argtypes = [ctypes.c_void_p, ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_int)]
        lib.tecdsa_modexp_batch.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p,
                                            ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p,
                                            ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int]
        lib.tecdsa_imad_peak.argtypes = [ctypes.c_void_p, ctypes.POINTER(ctypes.c_double), ctypes.POINTER(ctypes.c_float)]
        _lib = lib
    return _lib


# ----------------------------------------------------------------------------- limb packing
def ints_to_limbs(vals: Sequence[int], k: int) -> np.ndarray:
    """Python ints -> (len, k) uint32 little-endian limb rows (the ABI's operand-major layout)."""
    buf = b"".join(int(v).to_bytes(4 * k, "little") for v in vals)
    return np.frombuffer(buf, dtype="<u4").reshape(len(vals), k).copy()


def limbs_to_ints(a: np.ndarray) -> List[int]:
    a = np.ascontiguousarray(a, dtype="<u4")
    return [int.from_bytes(a[i].tobytes(), "little") for i in range(a.shape[0])]


def _ptr(a) -> Optional[int]:
    """Address of a numpy array (host) or torch tensor (host or device)."""
    if a is None:
        return None
    if isinstance(a, np.ndarray):
        assert a.flags["C_CONTIGUOUS"]
        return a.ctypes.data
    return a.data_ptr()            # torch.Tensor


class Engine:
    """One engine context = one GPU + one stream (tecdsa_ctx)."""

    def __init__(self, device: int = 0, stream: Optional[int] = None):
        self.lib = load_library()
        self._ctx = ctypes.c_void_p()
        rc = self.lib.tecdsa_ctx_create(ctypes.byref(self._ctx), device, stream)
        if rc != 0:
            raise EngineError(f"tecdsa_ctx_create: {self.lib.tecdsa_last_error().decode()} (rc={rc})")
        self.device = device

    def close(self):
        if self._ctx:
            self.lib.tecdsa_ctx_destroy(self._ctx)
            self._ctx = ctypes.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _ck(self, rc: int, what: str):
        if rc != 0:
            raise EngineError(f"{what}: {self.lib.tecdsa_last_error().decode()} (rc={rc})")

    def sync(self):
        self._ck(self.lib.tecdsa_ctx_sync(self._ctx), "sync")

    def set_tpi(self, mod_bits: int, tpi: int):
        self._ck(self.lib.tecdsa_ctx_set_tpi(self._ctx, mod_bits, tpi), "set_tpi")

    def set_option(self, name: str, value: int):
        self.lib.tecdsa_ctx_set_option.argtypes = [ctypes.c_void_p, ctypes.c_char_p, ctypes.c_int]
        self._ck(self.lib.tecdsa_ctx_set_option(self._ctx, name.encode(), value), "set_option")

    def last_kernel_ms(self):
        ms, n = ctypes.c_float(), ctypes.c_int()
        self._ck(self.lib.tecdsa_ctx_last_kernel_ms(self._ctx, ctypes.byref(ms), ctypes.byref(n)), "last_kernel_ms")
        return ms.value, n.value

    def launch_count(self) -> int:
        return int(self.lib.tecdsa_ctx_launch_count(self._ctx))

    def imad_peak(self, chained: bool = False):
        """(MAC32/s, ms) of the integer multiply-add saturation micro-benchmark: carry-free IMAD.WIDE.U32, or (chained) the
        IMAD.WIDE.U32.X carry chains the Montgomery rows are made of."""
        v, ms = ctypes.c_double(), ctypes.c_float()
        fn = self.lib.tecdsa_imad_peak_chained if chained else self.lib.tecdsa_imad_peak
        fn.argtypes = [ctypes.c_void_p, ctypes.POINTER(ctypes.c_double), ctypes.POINTER(ctypes.c_float)]
        self._ck(fn(self._ctx, ctypes.byref(v), ctypes.byref(ms)), "imad_peak")
        return v.value, ms.value

    # ---- BigInt::mod_pow, batched -------------------------------------------------------
    def modexp_raw(self, mod_bits: int, exp_limbs: int, base, exp, modulus, out, status=None, mod_idx=None,
                   n_mod: int = 0, count: Optional[int] = None, mem: int = HOST):
        """Direct ABI call on caller buffers (numpy for HOST, torch CUDA tensors for DEVICE)."""
        if count is None:
            count = base.shape[0]
        self._ck(self.lib.tecdsa_modexp_batch(self._ctx, mod_bits, exp_limbs, _ptr(base), _ptr(exp), _ptr(modulus),
                                              _ptr(mod_idx), n_mod, _ptr(out), _ptr(status), count, mem), "modexp_batch")

    def mod_pow(self, base: Iterable[int], exponent: Iterable[int], modulus: Iterable[int], mod_bits: int = 2048,
                exp_bits: Optional[int] = None):
        """Batched `BigInt::mod_pow(base, exponent, modulus)`; returns (results, status)."""
        base, exponent, modulus = list(base), list(exponent), list(modulus)
        n = len(base)
        if n == 0:
            return [], np.zeros(0, dtype=np.uint8)
        k = mod_bits // 32
        if exp_bits is None:
            exp_bits = max(1, max(int(e).bit_length() for e in exponent))
        el = (exp_bits + 31) // 32
        b, e, m = ints_to_limbs(base, k), ints_to_limbs(exponent, el), ints_to_limbs(modulus, k)
        out = np.zeros_like(b)
        st = np.full(n, 255, dtype=np.uint8)
        self.modexp_raw(mod_bits, el, b, e, m, out, st)
        return limbs_to_ints(out), st


# ----------------------------------------------------------------------------- L0 / L1 wrappers (batched BigInt / Paillier calls)
def _bind_l01(lib):
    if getattr(lib, "_l01_bound", False):
        return
    V, S, I = ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int
    lib.tecdsa_modmul_batch.argtypes = [V, I, V, V, V, V, S, V, S, I]
    lib.tecdsa_modinv_batch.argtypes = [V, I, V, V, V, S, V, V, S, I]
    lib.tecdsa_secp_mul_batch.argtypes = [V, V, V, V, S, I]
    lib.tecdsa_paillier_encrypt_batch.argtypes = [V, V, V, S, V, V, V, S, I]
    lib.tecdsa_paillier_mul_batch.argtypes = [V, V, V, S, V, V, I, V, S, I]
    lib.tecdsa_paillier_add_batch.argtypes = [V, V, V, S, V, V, V, S, I]
    lib.tecdsa_paillier_decrypt_batch.argtypes = [V, V, V, V, V, S, I]
    lib._l01_bound = True


def _mod_mul(self, a, b, modulus, mod_bits=2048):
    """Batched `BigInt::mod_mul(a, b, modulus)`."""
    _bind_l01(self.lib)
    k = mod_bits // 32
    A, B, M = ints_to_limbs(a, k), ints_to_limbs(b, k), ints_to_limbs(modulus, k)
    out = np.zeros_like(A)
    self._ck(self.lib.tecdsa_modmul_batch(self._ctx, mod_bits, _ptr(A), _ptr(B), _ptr(M), None, 0, _ptr(out), len(a), HOST), "modmul_batch")
    return limbs_to_ints(out)


def _mod_inv(self, a, modulus, mod_bits=2048):
    """Batched `BigInt::mod_inv(a, modulus)` -> list of int or None."""
    _bind_l01(self.lib)
    k = mod_bits // 32
    A, M = ints_to_limbs(a, k), ints_to_limbs(modulus, k)
    out = np.zeros_like(A)
    ok = np.zeros(len(a), dtype=np.uint8)
    self._ck(self.lib.tecdsa_modinv_batch(self._ctx, mod_bits, _ptr(A), _ptr(M), None, 0, _ptr(out), _ptr(ok), len(a), HOST), "modinv_batch")
    return [v if o else None for v, o in zip(limbs_to_ints(out), ok)]


def _secp_mul(self, points, scalars):
    """Batched `Point * Scalar`; points = None means the generator.  Points are (x, y) tuples or None (identity)."""
    _bind_l01(self.lib)
    n = len(scalars)
    K_ = ints_to_limbs(scalars, 8)
    P = None if points is None else ints_to_limbs([0 if p is None else p[0] | (p[1] << 256) for p in points], 16)
    out = np.zeros((n, 16), dtype=np.uint32)
    self._ck(self.lib.tecdsa_secp_mul_batch(self._ctx, _ptr(P), _ptr(K_), _ptr(out), n, HOST), "secp_mul_batch")
    return [None if v == 0 else (v & ((1 << 256) - 1), v >> 256) for v in limbs_to_ints(out)]


def _paillier_encrypt(self, n_list, key_idx, m, r):
    """`Paillier::encrypt_with_chosen_randomness` batched: c = (1 + m n) r^n mod n^2."""
    _bind_l01(self.lib)
    N, idx = ints_to_limbs(n_list, 64), np.asarray(key_idx, dtype=np.uint32)
    Mv, R = ints_to_limbs(m, 64), ints_to_limbs(r, 64)
    out = np.zeros((len(m), 128), dtype=np.uint32)
    self._ck(self.lib.tecdsa_paillier_encrypt_batch(self._ctx, _ptr(N), _ptr(idx), len(n_list), _ptr(Mv), _ptr(R), _ptr(out), len(m), HOST), "paillier_encrypt")
    return limbs_to_ints(out)


def _paillier_mul(self, n_list, key_idx, c, k, k_limbs=8):
    _bind_l01(self.lib)
    N, idx = ints_to_limbs(n_list, 64), np.asarray(key_idx, dtype=np.uint32)
    C, Kk = ints_to_limbs(c, 128), ints_to_limbs(k, k_limbs)
    out = np.zeros_like(C)
    self._ck(self.lib.tecdsa_paillier_mul_batch(self._ctx, _ptr(N), _ptr(idx), len(n_list), _ptr(C), _ptr(Kk), k_limbs, _ptr(out), len(c), HOST), "paillier_mul")
    return limbs_to_ints(out)


def _paillier_add(self, n_list, key_idx, c1, c2):
    _bind_l01(self.lib)
    N, idx = ints_to_limbs(n_list, 64), np.asarray(key_idx, dtype=np.uint32)
    C1, C2 = ints_to_limbs(c1, 128), ints_to_limbs(c2, 128)
    out = np.zeros_like(C1)
    self._ck(self.lib.tecdsa_paillier_add_batch(self._ctx, _ptr(N), _ptr(idx), len(n_list), _ptr(C1), _ptr(C2), _ptr(out), len(c1), HOST), "paillier_add")
    return limbs_to_ints(out)


def _paillier_decrypt(self, keysets_handle, key_rows, c):
    """`Paillier::decrypt` (CRT) batched over an uploaded key set (gg20.KeySets)."""
    _bind_l01(self.lib)
    rows = np.asarray(key_rows, dtype=np.uint32)
    C = ints_to_limbs(c, 128)
    out = np.zeros((len(c), 64), dtype=np.uint32)
    self._ck(self.lib.tecdsa_paillier_decrypt_batch(self._ctx, keysets_handle, _ptr(rows), _ptr(C), _ptr(out), len(c), HOST), "paillier_decrypt")
    return limbs_to_ints(out)


# ----------------------------------------------------------------------------- records, gather, profiling
REC_BYTES = 256
REC = {"status": (0, 1), "R": (1, 33), "sigma": (34, 32), "k": (66, 32), "t0": (98, 33), "t1": (131, 33), "digest": (164, 32)}   # (offset, bytes)


class _LaunchInfo(ctypes.Structure):
    _fields_ = [("kernel", ctypes.c_char * 48), ("ms", ctypes.c_float), ("mac32", ctypes.c_uint64)]


def _bind_rec(lib):
    if getattr(lib, "_rec_bound", False):
        return
    V, S, I = ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int
    lib.tecdsa_gg20_pack_records.argtypes = [V] * 7 + [S, V]
    lib.tecdsa_gather_results.argtypes = [V, V, V, S, V]
    lib.tecdsa_nccl_unique_id.argtypes = [V]
    lib.tecdsa_nccl_comm_create.argtypes = [V, V, I, I, ctypes.POINTER(V)]
    lib.tecdsa_nccl_comm_destroy.argtypes = [V]
    lib.tecdsa_gg20_offline_records.argtypes = [V, V, V, V, S, V, V, I]
    lib.tecdsa_ctx_work.argtypes = [V, ctypes.POINTER(ctypes.c_uint64), I]
    lib.tecdsa_ctx_profile.argtypes = [V, I]
    lib.tecdsa_ctx_profile_read.argtypes = [V, ctypes.POINTER(_LaunchInfo), S, ctypes.POINTER(S)]
    lib._rec_bound = True


def _work(self, reset: bool = False) -> int:
    """multiply-accumulates (32x32+64) executed by the big-integer kernels since the last reset (tecdsa_ctx_work)"""
    _bind_rec(self.lib)
    v = ctypes.c_uint64()
    self._ck(self.lib.tecdsa_ctx_work(self._ctx, ctypes.byref(v), 1 if reset else 0), "ctx_work")
    return int(v.value)


def _pack_records(self, status, R, sigma, t_vec, digest, rnd, n_units, records):
    _bind_rec(self.lib)
    self._ck(self.lib.tecdsa_gg20_pack_records(self._ctx, _ptr(status), _ptr(R), _ptr(sigma), _ptr(t_vec), _ptr(digest), _ptr(rnd), n_units, _ptr(records)), "pack_records")


def _gather_results(self, comm, records, n_units, all_records):
    _bind_rec(self.lib)
    self._ck(self.lib.tecdsa_gather_results(self._ctx, comm, _ptr(records), n_units, _ptr(all_records)), "gather_results")


def _nccl_unique_id(self) -> np.ndarray:
    _bind_rec(self.lib)
    out = np.zeros(128, dtype=np.uint8)
    self._ck(self.lib.tecdsa_nccl_unique_id(out.ctypes.data), "nccl_unique_id")
    return out


def _nccl_comm_create(self, uid: np.ndarray, nranks: int, rank: int):
    _bind_rec(self.lib)
    uid = np.ascontiguousarray(uid, dtype=np.uint8)
    comm = ctypes.c_void_p()
    self._ck(self.lib.tecdsa_nccl_comm_create(self._ctx, uid.ctypes.data, nranks, rank, ctypes.byref(comm)), "nccl_comm_create")
    return comm


def _nccl_comm_destroy(self, comm):
    _bind_rec(self.lib)
    self._ck(self.lib.tecdsa_nccl_comm_destroy(comm), "nccl_comm_destroy")


def _offline_records(self, keys, comm, sessions, n_sessions, rnd, all_records, mem=HOST):
    """tecdsa_gg20_offline_records: inputs -> Round0..6 -> 256-byte records -> gather -> (HOST) D2H, one call"""
    _bind_rec(self.lib)
    self._ck(self.lib.tecdsa_gg20_offline_records(self._ctx, keys.handle, comm, _ptr(sessions), n_sessions, _ptr(rnd), _ptr(all_records), mem), "gg20_offline_records")


def _profile_step(self, fn):
    """Run fn() once with per-launch CUDA-event profiling on -> {kernel: {"ms", "launches", "mac32"}}"""
    _bind_rec(self.lib)
    self._ck(self.lib.tecdsa_ctx_profile(self._ctx, 1), "ctx_profile")
    try:
        fn()
        n = ctypes.c_size_t()
        buf = (_LaunchInfo * 4096)()
        self._ck(self.lib.tecdsa_ctx_profile_read(self._ctx, buf, 4096, ctypes.byref(n)), "ctx_profile_read")
    finally:
        self.lib.tecdsa_ctx_profile(self._ctx, 0)
    out = {}
    for i in range(min(n.value, 4096)):
        e = out.setdefault(buf[i].kernel.decode(), {"ms": 0.0, "launches": 0, "mac32": 0})
        e["ms"] += float(buf[i].ms); e["launches"] += 1; e["mac32"] += int(buf[i].mac32)
    return out


Engine.work, Engine.pack_records, Engine.gather_results, Engine.offline_records = _work, _pack_records, _gather_results, _offline_records
Engine.nccl_unique_id, Engine.nccl_comm_create, Engine.nccl_comm_destroy, Engine.profile_step = _nccl_unique_id, _nccl_comm_create, _nccl_comm_destroy, _profile_step
# ----------------------------------------------------------------------------- Scalar / Point / BigInt helpers (L0)
def _bind_ec(lib):
    if getattr(lib, "_ec_bound", False):
        return
    V, S, I = ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int
    for n in ("add", "sub"):
        getattr(lib, f"tecdsa_secp_{n}_batch").argtypes = [V, V, V, V, S, I]
    lib.tecdsa_secp_compress_batch.argtypes = [V, V, V, S, I]
    lib.tecdsa_secp_decompress_batch.argtypes = [V, V, V, V, S, I]
    for n in ("mul", "add", "sub"):
        getattr(lib, f"tecdsa_secp_scalar_{n}_batch").argtypes = [V, V, V, V, S, I]
    lib.tecdsa_secp_scalar_inv_batch.argtypes = [V, V, V, V, S, I]
    lib.tecdsa_secp_scalar_from_bigint_batch.argtypes = [V, V, I, V, S, I]
    lib.tecdsa_wide_muladd_batch.argtypes = [V, V, I, V, I, V, I, V, I, S, I]
    lib.tecdsa_unit_mod_check_batch.argtypes = [V, I, V, V, V, S, V, S, I]
    lib.tecdsa_sha256_batch.argtypes = [V, V, V, V, S, I]
    lib._ec_bound = True


def _pack_pts(points):
    return ints_to_limbs([0 if p is None else p[0] | (p[1] << 256) for p in points], 16)


def _unpack_pts(arr):
    return [None if v == 0 else (v & ((1 << 256) - 1), v >> 256) for v in limbs_to_ints(arr)]


def _point_add(self, a, b, subtract=False):
    """Batched `Point + Point` / `Point - Point`; points are (x, y) tuples or None (identity)."""
    _bind_ec(self.lib)
    A, B = _pack_pts(a), _pack_pts(b)
    out = np.zeros_like(A)
    fn = self.lib.tecdsa_secp_sub_batch if subtract else self.lib.tecdsa_secp_add_batch
    self._ck(fn(self._ctx, _ptr(A), _ptr(B), _ptr(out), len(a), HOST), "secp_add/sub")
    return _unpack_pts(out)


def _point_compress(self, points):
    """Batched `Point::to_bytes(true)` -> list of 33-byte strings"""
    _bind_ec(self.lib)
    A = _pack_pts(points)
    out = np.zeros((len(points), 33), dtype=np.uint8)
    self._ck(self.lib.tecdsa_secp_compress_batch(self._ctx, _ptr(A), _ptr(out), len(points), HOST), "secp_compress")
    return [bytes(r) for r in out]


def _point_decompress(self, encodings):
    """Batched `Point::from_bytes` of 33-byte compressed encodings -> list of (x, y) or None (malformed)"""
    _bind_ec(self.lib)
    n = len(encodings)
    buf = np.frombuffer(b"".join(bytes(e).ljust(33, b"\0")[:33] for e in encodings), dtype=np.uint8).reshape(n, 33).copy()
    out, ok = np.zeros((n, 16), dtype=np.uint32), np.zeros(n, dtype=np.uint8)
    self._ck(self.lib.tecdsa_secp_decompress_batch(self._ctx, _ptr(buf), _ptr(out), _ptr(ok), n, HOST), "secp_decompress")
    return [p if o else None for p, o in zip(_unpack_pts(out), ok)]


def _scalar_op(self, op, a, b=None):
    """Batched `Scalar` arithmetic mod q: op in {"mul", "add", "sub", "inv"}; inv returns None for zero"""
    _bind_ec(self.lib)
    A = ints_to_limbs(a, 8)
    out = np.zeros_like(A)
    if op == "inv":
        ok = np.zeros(len(a), dtype=np.uint8)
        self._ck(self.lib.tecdsa_secp_scalar_inv_batch(self._ctx, _ptr(A), _ptr(out), _ptr(ok), len(a), HOST), "secp_scalar_inv")
        return [v if o else None for v, o in zip(limbs_to_ints(out), ok)]
    B = ints_to_limbs(b, 8)
    self._ck(getattr(self.lib, f"tecdsa_secp_scalar_{op}_batch")(self._ctx, _ptr(A), _ptr(B), _ptr(out), len(a), HOST), "secp_scalar_" + op)
    return limbs_to_ints(out)


def _scalar_from_bigint(self, x, limbs=64):
    _bind_ec(self.lib)
    X = ints_to_limbs(x, limbs)
    out = np.zeros((len(x), 8), dtype=np.uint32)
    self._ck(self.lib.tecdsa_secp_scalar_from_bigint_batch(self._ctx, _ptr(X), limbs, _ptr(out), len(x), HOST), "secp_scalar_from_bigint")
    return limbs_to_ints(out)


def _wide_muladd(self, a, b, c, a_limbs, b_limbs, c_limbs, out_limbs):
    """Batched exact a*b + c (no modulus).  out_limbs must hold the result for every operand value: out_limbs >=
    max(a_limbs + b_limbs, c_limbs) + 1, or out_limbs == a_limbs + b_limbs with c_limbs <= max(a_limbs, b_limbs); other
    widths raise EngineError (TECDSA_E_ARG)."""
    _bind_ec(self.lib)
    A, B, C = ints_to_limbs(a, a_limbs), ints_to_limbs(b, b_limbs), ints_to_limbs(c, c_limbs)
    out = np.zeros((len(a), out_limbs), dtype=np.uint32)
    self._ck(self.lib.tecdsa_wide_muladd_batch(self._ctx, _ptr(A), a_limbs, _ptr(B), b_limbs, _ptr(C), c_limbs, _ptr(out), out_limbs, len(a), HOST), "wide_muladd")
    return limbs_to_ints(out)


def _unit_mod_check(self, r, modulus, mod_bits=2048):
    """Batched acceptance test of `SampleFromMultiplicativeGroup`: r < N and gcd(r, N) == 1"""
    _bind_ec(self.lib)
    k = mod_bits // 32
    R, M = ints_to_limbs(r, k), ints_to_limbs(modulus, k)
    ok = np.zeros(len(r), dtype=np.uint8)
    self._ck(self.lib.tecdsa_unit_mod_check_batch(self._ctx, mod_bits, _ptr(R), _ptr(M), None, 0, _ptr(ok), len(r), HOST), "unit_mod_check")
    return [bool(x) for x in ok]


def _sha256(self, messages):
    """Batched SHA-256 of byte strings"""
    _bind_ec(self.lib)
    n = len(messages)
    offs = np.zeros(n + 1, dtype=np.uint64)
    offs[1:] = np.cumsum([len(m) for m in messages])
    blob = np.frombuffer(b"".join(messages) or b"\0", dtype=np.uint8).copy()
    out = np.zeros((n, 32), dtype=np.uint8)
    self._ck(self.lib.tecdsa_sha256_batch(self._ctx, _ptr(blob), _ptr(offs), _ptr(out), n, HOST), "sha256")
    return [bytes(r) for r in out]


def seed_words(seed: bytes) -> np.ndarray:
    """a 32-byte seed as the 8 little-endian words the ABI takes"""
    if len(seed) != 32:
        raise ValueError("the sampler's seed is 32 bytes")
    return np.frombuffer(bytes(seed), dtype="<u4").copy()


def _sample(self, kind: int, count: int, seed: bytes, stream: int = 0, first_id: int = 0, bound=None, bound_idx=None, bits: int = 0,
            limbs: Optional[int] = None):
    """Batched seeded sampling (tecdsa_sample_batch): element i = one value of `kind` (SAMPLE_*) on `stream` for element id
    first_id + i.  bound = list of ints, one per element, or a table that bound_idx[i] indexes.  -> (values, status); a value whose
    status is ST_SAMPLING is 0.  A (seed, stream, element id) triple must never be used twice."""
    lib = self.lib
    if not getattr(lib, "_sample_bound", False):
        V, S, I = ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int
        lib.tecdsa_sample_batch.argtypes = [V, V, ctypes.c_uint64, ctypes.c_uint32, I, I, V, V, S, I, V, V, S, I]
        lib._sample_bound = True
    bounded = kind in (SAMPLE_BELOW, SAMPLE_UNIT, SAMPLE_RANGE1)
    if limbs is None:
        width = 256 if kind == SAMPLE_SCALAR else bits if kind == SAMPLE_BITS else max([int(b).bit_length() for b in bound] + [1])
        limbs = (width + 127) // 128 * 4
    B = ints_to_limbs(bound, limbs) if bounded else None
    idx = None if bound_idx is None or not bounded else np.asarray(bound_idx, dtype=np.uint32)
    out = np.zeros((count, limbs), dtype=np.uint32)
    st = np.full(count, 255, dtype=np.uint8)
    sw = seed_words(seed)
    try:
        self._ck(lib.tecdsa_sample_batch(self._ctx, _ptr(sw), first_id, stream, kind, bits, _ptr(B), _ptr(idx), 0 if B is None else B.shape[0], limbs,
                                         _ptr(out), _ptr(st), count, HOST), "sample_batch")
    finally:
        sw[:] = 0
    return limbs_to_ints(out), st


Engine.sample = _sample
Engine.point_add, Engine.point_compress, Engine.point_decompress, Engine.scalar_op = _point_add, _point_compress, _point_decompress, _scalar_op
Engine.scalar_from_bigint, Engine.wide_muladd, Engine.unit_mod_check, Engine.sha256 = _scalar_from_bigint, _wide_muladd, _unit_mod_check, _sha256
Engine.mod_mul, Engine.mod_inv, Engine.secp_mul = _mod_mul, _mod_inv, _secp_mul
Engine.paillier_encrypt, Engine.paillier_mul, Engine.paillier_add, Engine.paillier_decrypt = _paillier_encrypt, _paillier_mul, _paillier_add, _paillier_decrypt
