/* tecdsa_b200 — C ABI of the batched threshold-ECDSA arithmetic engine (H100, sm_90a).
 *
 * The reference (ZenGo-X/multi-party-ecdsa @ 7d8bd41) has no FFI of its own: its seam is
 * the Rust trait surface of curv-kzen `BigInt`, `Scalar/Point<Secp256k1>`, kzen-paillier
 * `Paillier::*` and the in-tree proof structs.  Every entry point below is the BATCHED form
 * of one of those scalar calls and cites the reference call site it replaces (paths are
 * relative to /root/reference).  INTEGRATION.md shows the Rust `extern "C"` shim a maintainer
 * would add so that the protocol modules under src/protocols link against this library.
 *
 * Conventions
 *   - Big integers are little-endian arrays of uint32_t limbs, operand-major:
 *     x[i*K .. i*K+K) is operand i (K = bits/32).  Rows must be 16-byte aligned.
 *     Byte strings (hash inputs, compressed points) are big-endian exactly as
 *     `BigInt::to_bytes()` / `Point::to_bytes(true)` produce them.
 *   - `mem` says where caller buffers live: TECDSA_HOST (library stages H2D/D2H on the
 *     context stream) or TECDSA_DEVICE (pointers are device pointers, nothing is copied).
 *   - Every call returns 0 on success, <0 on API/CUDA failure (tecdsa_last_error()).
 *     Per-element outcomes go to `status[count]` (TECDSA_ST_*); a failed element never
 *     aborts the batch and never panics, unlike the reference's assert!/unwrap() sites.
 *   - Calls are asynchronous on the context's stream for TECDSA_DEVICE, synchronous for
 *     TECDSA_HOST.  A context is not thread-safe; distinct contexts are independent.
 *   - No randomness is drawn inside the library: every sampled value of the reference
 *     (`BigInt::sample_below`, `Scalar::random`) is an explicit input.
 */
#ifndef TECDSA_B200_H
#define TECDSA_B200_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct tecdsa_ctx tecdsa_ctx;
typedef struct tecdsa_keyset tecdsa_keyset;   /* device-resident key material, see tecdsa_keys_upload */

enum { TECDSA_HOST = 0, TECDSA_DEVICE = 1 };

/* return codes */
enum { TECDSA_OK = 0, TECDSA_E_ARG = -1, TECDSA_E_CUDA = -2, TECDSA_E_NOMEM = -3, TECDSA_E_UNSUPPORTED = -4 };

/* per-element status bytes; numbering follows the reference's failure points */
enum {
    TECDSA_ST_OK = 0,
    TECDSA_ST_EVEN_MODULUS = 1,   /* mod_pow on an even modulus: outside Montgomery domain  */
    TECDSA_ST_INVALID_KEY = 2,    /* Error::InvalidKey           src/utilities/mta/mod.rs:120,130,177 */
    TECDSA_ST_RANGE = 3,          /* s1 > q^3                    src/utilities/mta/range_proofs.rs:118 */
    TECDSA_ST_NOT_INVERTIBLE = 4, /* mod_inv -> None             range_proofs.rs:123-127,136-139; zk_pdl_with_slack/mod.rs:192 */
    TECDSA_ST_HASH_MISMATCH = 5,  /* e != self.e                 range_proofs.rs:151 */
    TECDSA_ST_PDL_VERIFY = 6,     /* ZkPdlWithSlackError::Verify zk_pdl_with_slack/mod.rs:177 */
    TECDSA_ST_PHASE5_BAD_SUM = 7, /* Error::Phase5BadSum         gg_2020/party_i.rs:774 */
    TECDSA_ST_PHASE6 = 8,         /* Error::Phase6Error          gg_2020/party_i.rs:846 */
    TECDSA_ST_INVALID_SIG = 9,    /* Error::InvalidSig           gg_2020/party_i.rs:908,934 */
    TECDSA_ST_PROOF = 10,         /* a curv sigma proof (DLog/Pedersen/HomoElGamal) failed to verify */
    TECDSA_ST_COMMITMENT = 11,    /* "bad gamma_i decommit"      gg_2020/party_i.rs:650-674 */
    TECDSA_ST_INVALID_SS = 12     /* Error::InvalidSS            gg_2018/party_i.rs:262-281 (reported by the host-composed key-generation drivers) */
};

/* ---- context ------------------------------------------------------------------------ */
/* `stream` is the cudaStream_t every launch and copy of this context goes to (NULL = the
 * device's default stream, which is also torch's default current stream).                  */
int tecdsa_ctx_create(tecdsa_ctx** ctx, int device, void* stream);
int tecdsa_ctx_destroy(tecdsa_ctx* ctx);
int tecdsa_ctx_sync(tecdsa_ctx* ctx);
const char* tecdsa_last_error(void);
/* Lane-group width (4, 8, 16 or 32 lanes per operand; 32 = one warp per operand) used for
 * `mod_bits`-wide moduli.  0 restores the tuned default. */
int tecdsa_ctx_set_tpi(tecdsa_ctx* ctx, int mod_bits, int tpi);
/* Named tuning options (results never depend on them).  "sqr" = 1: tecdsa_modexp_batch squares through the block-partitioned
 * Montgomery squaring of csrc/sqr.cuh (fewer multiply-accumulates, but slower: off by default).                             */
int tecdsa_ctx_set_option(tecdsa_ctx* ctx, const char* name, int value);
/* Device time (ms, CUDA events on the context stream) of the kernels of the last call and
 * how many kernels that call launched. */
int tecdsa_ctx_last_kernel_ms(tecdsa_ctx* ctx, float* ms, int* launches);
/* Total kernels launched through this context since creation. */
uint64_t tecdsa_ctx_launch_count(tecdsa_ctx* ctx);

/* ---- L0: big-integer arithmetic --------------------------------------------------------
 * out[i] = base[i] ^ exp[i] mod modulus[i]            (BigInt::mod_pow -> GMP mpz_powm;
 *   call sites src/utilities/mta/range_proofs.rs:52,54,57,86,122,129,130,135,141;
 *   src/utilities/zk_pdl_with_slack/mod.rs:189,193,196)
 * mod_bits in {1024, 2048, 4096}; operands are K = mod_bits/32 limbs; the modulus must be
 * odd (else TECDSA_ST_EVEN_MODULUS and a zero output); base may be any K-limb value (it is
 * reduced); exp is `exp_limbs` limbs (the batch's public maximum width, zero-padded).
 * If mod_idx != NULL, operand i uses modulus[mod_idx[i]] out of `n_mod` rows, else row i.  */
int tecdsa_modexp_batch(tecdsa_ctx* ctx, int mod_bits, int exp_limbs, const uint32_t* base, const uint32_t* exp,
                        const uint32_t* modulus, const uint32_t* mod_idx, size_t n_mod, uint32_t* out,
                        uint8_t* status, size_t count, int mem);

/* out[i] = a[i] * b[i] mod modulus   (BigInt::mod_mul, src/utilities/zk_pdl_with_slack/mod.rs:198; the `(x * y) % n`
 * products of src/utilities/mta/range_proofs.rs:52-57,129-141).  mod_bits in {2048, 4096}, odd moduli.            */
int tecdsa_modmul_batch(tecdsa_ctx* ctx, int mod_bits, const uint32_t* a, const uint32_t* b, const uint32_t* modulus,
                        const uint32_t* mod_idx, size_t n_mod, uint32_t* out, size_t count, int mem);
/* out[i] = a[i]^-1 mod modulus, ok[i] = 1; or ok[i] = 0 (and out = 0) when gcd != 1 — `BigInt::mod_inv -> Option`
 * (src/utilities/mta/range_proofs.rs:122,135; src/utilities/zk_pdl_with_slack/mod.rs:192).  Odd moduli.            */
int tecdsa_modinv_batch(tecdsa_ctx* ctx, int mod_bits, const uint32_t* a, const uint32_t* modulus, const uint32_t* mod_idx,
                        size_t n_mod, uint32_t* out, uint8_t* ok, size_t count, int mem);
/* out[i] = scalars[i] * points[i] on secp256k1 (`Point * Scalar`, gg_2020/party_i.rs:560-562,682,784); points == NULL
 * means the generator (`Point::generator() * s`).  Points are affine x||y (16 limbs, all-zero = identity); scalars
 * are reduced mod q; a point that is not on the curve yields the identity.                                          */
int tecdsa_secp_mul_batch(tecdsa_ctx* ctx, const uint32_t* points, const uint32_t* scalars, uint32_t* out, size_t count, int mem);

/* ---- L0: the rest of the Scalar<Secp256k1> / Point<Secp256k1> / BigInt surface src/ calls between the heavy steps ----------
 * Points are affine x||y (16 limbs, all-zero = identity), scalars 8 limbs reduced mod q on entry.
 * secp_add / secp_sub: `Point + Point`, `Point - Point` (gg_2020/party_i.rs:771-772,839-840).
 * secp_compress: `Point::to_bytes(true)` -> 33 bytes per point (party_i.rs:577-580; zk_pdl_with_slack/mod.rs:102-110); the
 *   identity gives 33 zero bytes.  secp_decompress: `Point::from_bytes` of such an encoding; ok = 0 (and the identity) for a
 *   malformed one (bad prefix, x >= p, x^3 + 7 a non-residue).
 * secp_scalar_{mul,add,sub,inv}: `Scalar * + - invert()` (party_i.rs:599-617,635-640,857-863); inv: ok = 0 for zero.
 * secp_scalar_from_bigint: `Scalar::from(&BigInt)` — a `limbs`-limb integer reduced mod q (mta/mod.rs:132,166).
 * wide_muladd: a*b + c over the integers, no modulus (`e * a + alpha`, `e * rho + gamma`; mta/range_proofs.rs:87-88):
 *   out_limbs >= a_limbs + b_limbs and > c_limbs.
 * unit_mod_check: the acceptance test of `SampleFromMultiplicativeGroup::from_modulo / from_paillier_key`
 *   (mta/range_proofs.rs:538-557): ok = 1 iff r < N and gcd(r, N) = 1 (odd N; mod_bits 2048 or 4096) — the caller's sampling
 *   loop draws again where ok = 0, exactly as the reference's `while r.gcd(N) != 1`.
 * sha256: SHA-256 of arbitrary byte strings, message i = bytes[offsets[i], offsets[i+1]) -> digests [count][32]
 *   (TECDSA_HOST only: the offsets are read on the host).                                                                */
int tecdsa_secp_add_batch(tecdsa_ctx* ctx, const uint32_t* a, const uint32_t* b, uint32_t* out, size_t count, int mem);
int tecdsa_secp_sub_batch(tecdsa_ctx* ctx, const uint32_t* a, const uint32_t* b, uint32_t* out, size_t count, int mem);
int tecdsa_secp_compress_batch(tecdsa_ctx* ctx, const uint32_t* points, uint8_t* out33, size_t count, int mem);
int tecdsa_secp_decompress_batch(tecdsa_ctx* ctx, const uint8_t* in33, uint32_t* points, uint8_t* ok, size_t count, int mem);
int tecdsa_secp_scalar_mul_batch(tecdsa_ctx* ctx, const uint32_t* a, const uint32_t* b, uint32_t* out, size_t count, int mem);
int tecdsa_secp_scalar_add_batch(tecdsa_ctx* ctx, const uint32_t* a, const uint32_t* b, uint32_t* out, size_t count, int mem);
int tecdsa_secp_scalar_sub_batch(tecdsa_ctx* ctx, const uint32_t* a, const uint32_t* b, uint32_t* out, size_t count, int mem);
int tecdsa_secp_scalar_inv_batch(tecdsa_ctx* ctx, const uint32_t* a, uint32_t* out, uint8_t* ok, size_t count, int mem);
int tecdsa_secp_scalar_from_bigint_batch(tecdsa_ctx* ctx, const uint32_t* x, int limbs, uint32_t* out, size_t count, int mem);
int tecdsa_wide_muladd_batch(tecdsa_ctx* ctx, const uint32_t* a, int a_limbs, const uint32_t* b, int b_limbs, const uint32_t* c, int c_limbs,
                             uint32_t* out, int out_limbs, size_t count, int mem);
int tecdsa_unit_mod_check_batch(tecdsa_ctx* ctx, int mod_bits, const uint32_t* r, const uint32_t* modulus, const uint32_t* mod_idx, size_t n_mod,
                                uint8_t* ok, size_t count, int mem);
int tecdsa_sha256_batch(tecdsa_ctx* ctx, const uint8_t* bytes, const uint64_t* offsets, uint8_t* digests, size_t count, int mem);

/* ---- L1: Paillier (kzen-paillier 0.4.2 as called from src/utilities/mta/mod.rs:68,133,140,145,165) ----------------
 * n = [n_keys][64] public moduli, key_idx[i] selects the key of element i (NULL: element i uses row i).
 * encrypt: c = (1 + m n) r^n mod n^2 (`encrypt_with_chosen_randomness`); mul: c^k mod n^2 (k has k_limbs <= 64 limbs);
 * add: c1 c2 mod n^2; decrypt: CRT form over an uploaded key set (row = keyset*3 + party), m in [0, n).              */
int tecdsa_paillier_encrypt_batch(tecdsa_ctx* ctx, const uint32_t* n, const uint32_t* key_idx, size_t n_keys, const uint32_t* m,
                                  const uint32_t* r, uint32_t* c, size_t count, int mem);
int tecdsa_paillier_mul_batch(tecdsa_ctx* ctx, const uint32_t* n, const uint32_t* key_idx, size_t n_keys, const uint32_t* c,
                              const uint32_t* k, int k_limbs, uint32_t* out, size_t count, int mem);
int tecdsa_paillier_add_batch(tecdsa_ctx* ctx, const uint32_t* n, const uint32_t* key_idx, size_t n_keys, const uint32_t* c1,
                              const uint32_t* c2, uint32_t* out, size_t count, int mem);
int tecdsa_paillier_decrypt_batch(tecdsa_ctx* ctx, const tecdsa_keyset* ks, const uint32_t* key_row, const uint32_t* c,
                                  uint32_t* m, size_t count, int mem);

/* ---- L2: MtA range proof, Alice side (src/utilities/mta/range_proofs.rs:105-193) ---------------------------------
 * ek_row / st_row: key rows (keyset*3 + party) of Alice's Paillier key and of the verifier's (N~, h1, h2) statement.
 * generate: a (8 limbs), cipher (128), r (64) and the sampled alpha (24) < q^3, beta (64) in Z*_N, gamma (88) < q^3 N~,
 * rho (72) < q N~  ->  z (64), e (8), s (64), s1 (28), s2 (92).  verify: status[i] = TECDSA_ST_OK or the first failing
 * check (RANGE: s1 > q^3; NOT_INVERTIBLE; HASH_MISMATCH), i.e. `false` of AliceProof::verify.                         */
int tecdsa_alice_proof_generate_batch(tecdsa_ctx* ctx, const tecdsa_keyset* ks, const uint32_t* ek_row, const uint32_t* st_row,
                                      const uint32_t* a, const uint32_t* cipher, const uint32_t* r, const uint32_t* alpha,
                                      const uint32_t* beta, const uint32_t* gamma, const uint32_t* rho, uint32_t* z, uint32_t* e,
                                      uint32_t* s, uint32_t* s1, uint32_t* s2, size_t count, int mem);
int tecdsa_alice_proof_verify_batch(tecdsa_ctx* ctx, const tecdsa_keyset* ks, const uint32_t* ek_row, const uint32_t* st_row,
                                    const uint32_t* cipher, const uint32_t* z, const uint32_t* e, const uint32_t* s,
                                    const uint32_t* s1, const uint32_t* s2, uint8_t* status, size_t count, int mem);

/* ---- L2: PDL with slack (src/utilities/zk_pdl_with_slack/mod.rs:68-179) --------------------------------------
 * Statement (cipher, ek = key row ek_row, Q, G, (h1,h2,N~) = key row st_row); witness x (8 limbs), r (64).
 * prove: sampled alpha (24) < q^3, beta (64) in [1,N-1), rho (72) < q N~, gamma (88) < q^3 N~
 *        -> z (64), u1 (point, 16), u2 (128), u3 (64), s1 (28), s2 (64), s3 (92).
 * verify: status TECDSA_ST_OK or TECDSA_ST_PDL_VERIFY (incl. the reference's unwrap() panic on a non-invertible
 * z or ciphertext, mod.rs:192).                                                                                  */
int tecdsa_pdl_prove_batch(tecdsa_ctx* ctx, const tecdsa_keyset* ks, const uint32_t* ek_row, const uint32_t* st_row, const uint32_t* x,
                           const uint32_t* r, const uint32_t* cipher, const uint32_t* Q, const uint32_t* G, const uint32_t* alpha,
                           const uint32_t* beta, const uint32_t* rho, const uint32_t* gamma, uint32_t* z, uint32_t* u1, uint32_t* u2,
                           uint32_t* u3, uint32_t* s1, uint32_t* s2, uint32_t* s3, size_t count, int mem);
int tecdsa_pdl_verify_batch(tecdsa_ctx* ctx, const tecdsa_keyset* ks, const uint32_t* ek_row, const uint32_t* st_row, const uint32_t* cipher,
                            const uint32_t* Q, const uint32_t* G, const uint32_t* z, const uint32_t* u1, const uint32_t* u2,
                            const uint32_t* u3, const uint32_t* s1, const uint32_t* s2, const uint32_t* s3, uint8_t* status, size_t count, int mem);

/* ---- L2: Bob's MtA / MtAwc range proof (src/utilities/mta/range_proofs.rs:214-535; not called by OfflineStage,
 * part of the public proof surface).  generate: a_enc, mta_enc (128), b (8), beta_prim (64), r (64) and the sampled
 * alpha (24) < q^3, beta (64) in Z*_N, gamma (80) < q^2 N, ro (72) < q N~, ro_prim (88) < q^3 N~, sigma (72) < q N~,
 * tau (88) < q^3 N~  ->  t, z (64), e (8), s (64), s1 (28), s2 (92), t1 (84), t2 (92) and, when check != 0 (MtAwc,
 * `BobProofExt`), u = G * alpha (16).  verify: X == u == NULL is `BobProof::verify(.., None)`; otherwise
 * `BobProofExt::verify` with X = G * b.  status: OK / RANGE / NOT_INVERTIBLE / HASH_MISMATCH / PROOF (EC check). */
int tecdsa_bob_proof_generate_batch(tecdsa_ctx* ctx, const tecdsa_keyset* ks, const uint32_t* ek_row, const uint32_t* st_row, int check,
                                    const uint32_t* a_enc, const uint32_t* mta_enc, const uint32_t* b, const uint32_t* beta_prim,
                                    const uint32_t* r, const uint32_t* alpha, const uint32_t* beta, const uint32_t* gamma,
                                    const uint32_t* ro, const uint32_t* ro_prim, const uint32_t* sigma, const uint32_t* tau,
                                    uint32_t* t, uint32_t* z, uint32_t* e, uint32_t* s, uint32_t* s1, uint32_t* s2, uint32_t* t1,
                                    uint32_t* t2, uint32_t* u, size_t count, int mem);
int tecdsa_bob_proof_verify_batch(tecdsa_ctx* ctx, const tecdsa_keyset* ks, const uint32_t* ek_row, const uint32_t* st_row, const uint32_t* a_enc,
                                  const uint32_t* mta_out, const uint32_t* t, const uint32_t* z, const uint32_t* e, const uint32_t* s,
                                  const uint32_t* s1, const uint32_t* s2, const uint32_t* t1, const uint32_t* t2, const uint32_t* X,
                                  const uint32_t* u, uint8_t* status, size_t count, int mem);

/* ---- L2: the MtA share conversion messages (src/utilities/mta/mod.rs:52-179) ----------------------------------
 * message_a = `MessageA::a_with_predefined_randomness`: c = Enc(ek_row; a, r) and one AliceProof per statement;
 *   per-proof arrays are indexed [instance][statement] (n_st statements per instance, st_rows gives their key rows;
 *   n_st = 0 is the "no range proofs" form used by GG18 / blame).
 * message_b = `MessageB::b_with_predefined_randomness`: verifies every range proof of MessageA (any failure ->
 *   status TECDSA_ST_INVALID_KEY, like Err(InvalidKey)), c_b = c_a^b * Enc(beta'; r') mod N^2, beta = -beta' mod q,
 *   and the DLogProofs of b and beta' (40 limbs each, layout as tecdsa_dlog_prove_batch).
 * get_alpha = `MessageB::verify_proofs_get_alpha`: alpha' = Dec(dk_row; c_b) (64 limbs, optional output),
 *   alpha = alpha' mod q, status OK iff both DLogProofs verify and G*alpha == B*a + B'.                            */
int tecdsa_mta_message_a_batch(tecdsa_ctx* ctx, const tecdsa_keyset* ks, const uint32_t* ek_row, const uint32_t* st_rows, int n_st,
                               const uint32_t* a, const uint32_t* r, const uint32_t* alpha, const uint32_t* beta, const uint32_t* gamma,
                               const uint32_t* rho, uint32_t* c, uint32_t* z, uint32_t* e, uint32_t* s, uint32_t* s1, uint32_t* s2,
                               size_t count, int mem);
int tecdsa_mta_message_b_batch(tecdsa_ctx* ctx, const tecdsa_keyset* ks, const uint32_t* ek_row, const uint32_t* st_rows, int n_st,
                               const uint32_t* b, const uint32_t* c_a, const uint32_t* z, const uint32_t* e, const uint32_t* s,
                               const uint32_t* s1, const uint32_t* s2, const uint32_t* randomness, const uint32_t* beta_tag,
                               const uint32_t* nonce_b, const uint32_t* nonce_beta, uint32_t* c_b, uint32_t* b_proof,
                               uint32_t* beta_tag_proof, uint32_t* beta, uint8_t* status, size_t count, int mem);
int tecdsa_mta_get_alpha_batch(tecdsa_ctx* ctx, const tecdsa_keyset* ks, const uint32_t* dk_row, const uint32_t* a, const uint32_t* c_b,
                               const uint32_t* b_proof, const uint32_t* beta_tag_proof, uint32_t* alpha, uint32_t* alpha_plain,
                               uint8_t* status, size_t count, int mem);

/* ---- key-generation path (SURVEY.md section 8(f) rank 1) -----------------------------------------------------------
 * The checks one party runs on every other party's KeyGenBroadcastMessage1 / shares (gg_2020/party_i.rs:260-320, 322-367)
 * and the proofs it produces for its own (party_i.rs:137-156, 219-258, 313); proof bodies are zk-paillier 0.4.3 / curv 0.9
 * [R].  status: TECDSA_ST_OK / _PROOF (verifiers), _NOT_INVERTIBLE (provers).
 * correct_key_verify: `NiCorrectKeyProof::verify(&ek, salt)` (party_i.rs:288-291): n = [count][64], sigma = [count][11][64],
 *   salt = salt_len raw bytes (zk-paillier SALT_STRING = "KZen"); includes gcd(P, n) == 1 for the primorial P of all primes
 *   <= 6379 (an n with a small prime factor is rejected even when every sigma^n == rho holds);
 * composite_dlog_verify: `CompositeDLogProof::verify(&DLogStatement{N, g, ni})` (party_i.rs:296-303): x = [count][64],
 *   y = [count][y_limbs] (an integer, not reduced);
 * vss_validate_share: `VerifiableSS::validate_share(&share, index)` (party_i.rs:337-339): commitments =
 *   [count][n_commitments][16] affine points (coefficient 0 first), share = [count][8], index = [count].            */
int tecdsa_correct_key_verify_batch(tecdsa_ctx* ctx, const uint32_t* n, const uint32_t* sigma, const uint8_t* salt, int salt_len,
                                    uint8_t* status, size_t count, int mem);
int tecdsa_composite_dlog_verify_batch(tecdsa_ctx* ctx, const uint32_t* n_tilde, const uint32_t* g, const uint32_t* ni, const uint32_t* x,
                                       const uint32_t* y, int y_limbs, uint8_t* status, size_t count, int mem);
int tecdsa_vss_validate_share_batch(tecdsa_ctx* ctx, const uint32_t* commitments, int n_commitments, const uint32_t* share,
                                    const uint32_t* index, uint8_t* status, size_t count, int mem);
/* correct_key_prove: `NiCorrectKeyProof::proof(&dk, None)` (party_i.rs:225): p, q = [count][32] -> sigma [count][11][64]
 *   (sigma_j = rho_j^(N^-1 mod phi(N)) mod N);
 * composite_dlog_prove: `CompositeDLogProof::prove(&statement, &secret)` (party_i.rs:238-241): nonce r = [count][16]
 *   (< 2^512, the reference samples it), secret = [count][secret_limbs] -> x [count][64], y = r + e*secret [count][y_limbs],
 *   y_limbs >= secret_limbs + 9 and a multiple of 4;
 * vss_share: `VerifiableSS::share(t, n, &secret)` (party_i.rs:313) with explicit polynomial coefficients [count][t+1][8]
 *   (coefficient 0 = the secret) -> shares f(1..n) [count][n][8], commitments a_j*G [count][t+1][16];
 * h1_h2_n_tilde: `generate_h1_h2_N_tilde` (party_i.rs:137-156) with explicit samples: p~, q~ = [count][32], h1, xhi =
 *   [count][64] -> N~, h2 = h1^xhi, phi - xhi, phi - xhi^-1 (all [count][64]); NOT_INVERTIBLE where the reference's
 *   sampling loop would draw xhi again.                                                                              */
int tecdsa_correct_key_prove_batch(tecdsa_ctx* ctx, const uint32_t* p, const uint32_t* q, const uint8_t* salt, int salt_len,
                                   uint32_t* sigma, uint8_t* status, size_t count, int mem);
int tecdsa_composite_dlog_prove_batch(tecdsa_ctx* ctx, const uint32_t* n_tilde, const uint32_t* g, const uint32_t* ni, const uint32_t* secret,
                                      int secret_limbs, const uint32_t* r, uint32_t* x, uint32_t* y, int y_limbs, size_t count, int mem);
int tecdsa_vss_share_batch(tecdsa_ctx* ctx, int t, int n_shares, const uint32_t* coefficients, uint32_t* shares, uint32_t* commitments,
                           size_t count, int mem);
int tecdsa_h1_h2_n_tilde_batch(tecdsa_ctx* ctx, const uint32_t* p_t, const uint32_t* q_t, const uint32_t* h1, const uint32_t* xhi,
                               uint32_t* n_tilde, uint32_t* h2, uint32_t* xhi_neg, uint32_t* xhi_inv_neg, uint8_t* status, size_t count, int mem);

/* ---- identifiable abort (SURVEY.md section 8(f) rank 3; gg_2020/blame.rs) ------------------------------------------------
 * paillier_open: `Paillier::open(dk, c)` (blame.rs:252-256) over an uploaded key set: m = Dec(c) [count][64] and the
 *   randomness r [count][64] with c = (1 + m N) r^N mod N^2 (r = (c mod N)^(N^-1 mod phi(N)) mod N).
 * ecddh_prove / ecddh_verify: curv `ECDDHProof` [R] for statements (g1, h1 = x g1, g2, h2 = x g2) (blame.rs:258-271,405-417):
 *   proof = a1 16 | a2 16 | z 8 (40 limbs), nonce = the sampled s; status TECDSA_ST_OK / _PROOF.
 * The blame procedures (`phase5_blame`, `phase6_blame`, `phase7_blame`) re-derive every opened value with these and the
 * L0/L1 batch calls: multi-party-ecdsa_b200/blame.py.                                                                    */
int tecdsa_paillier_open_batch(tecdsa_ctx* ctx, const tecdsa_keyset* ks, const uint32_t* key_row, const uint32_t* c, uint32_t* m, uint32_t* r,
                               size_t count, int mem);
int tecdsa_ecddh_prove_batch(tecdsa_ctx* ctx, const uint32_t* x, const uint32_t* g1, const uint32_t* h1, const uint32_t* g2, const uint32_t* h2,
                             const uint32_t* nonce, uint32_t* proof, size_t count, int mem);
int tecdsa_ecddh_verify_batch(tecdsa_ctx* ctx, const uint32_t* proof, const uint32_t* g1, const uint32_t* h1, const uint32_t* g2, const uint32_t* h2,
                              uint8_t* status, size_t count, int mem);

/* ---- curv-kzen sigma proofs and hashes used by the protocol (out-of-tree crate; call sites cited) ----------------
 * Scalars are 8 limbs (reduced mod q on entry), points affine x||y 16 limbs.  Verifiers write TECDSA_ST_OK or
 * TECDSA_ST_PROOF.  Encodings [R]: challenges hash 65-byte uncompressed points and reduce the digest mod q.
 * DLogProof (mta/mod.rs:147-148,170-171): proof = pk 16 | pk_t_rand_commitment 16 | challenge_response 8 (40 limbs).
 * PedersenProof (party_i.rs:631, sign/rounds.rs:371-378): com = m G + r H (H = base_point2);
 *   proof = e 8 | a1 16 | a2 16 | z1 8 | z2 8 | pad 8 (64 limbs).
 * HomoELGamalProof (party_i.rs:778-833) for the statement (G, H = base_point2, Y = generator, D, E), witness (x, r):
 *   proof = T 16 | A3 16 | z1 8 | z2 8 (48 limbs).                                                                  */
int tecdsa_dlog_prove_batch(tecdsa_ctx* ctx, const uint32_t* sk, const uint32_t* nonce, uint32_t* proof, size_t count, int mem);
int tecdsa_dlog_verify_batch(tecdsa_ctx* ctx, const uint32_t* proof, uint8_t* status, size_t count, int mem);
int tecdsa_pedersen_prove_batch(tecdsa_ctx* ctx, const uint32_t* m, const uint32_t* r, const uint32_t* s1, const uint32_t* s2,
                                uint32_t* com, uint32_t* proof, size_t count, int mem);
int tecdsa_pedersen_verify_batch(tecdsa_ctx* ctx, const uint32_t* com, const uint32_t* proof, uint8_t* status, size_t count, int mem);
int tecdsa_heg_prove_batch(tecdsa_ctx* ctx, const uint32_t* G, const uint32_t* D, const uint32_t* E, const uint32_t* x, const uint32_t* r,
                           const uint32_t* s1, const uint32_t* s2, uint32_t* proof, size_t count, int mem);
int tecdsa_heg_verify_batch(tecdsa_ctx* ctx, const uint32_t* G, const uint32_t* D, const uint32_t* E, const uint32_t* proof, uint8_t* status,
                            size_t count, int mem);
/* `Sha256::new().chain_bigint(x_0)...chain_bigint(x_{k-1}).result_bigint()` (curv DigestExt; range_proofs.rs:143-150,
 * zk_pdl_with_slack/mod.rs:102-110): element i is n_items integers packed back to back, item j having item_limbs[j]
 * limbs; each is hashed as its minimal big-endian magnitude; digest = 8 limbs of the 256-bit result.  item_limbs is a
 * HOST array.                                                                                                        */
int tecdsa_sha256_bigints_batch(tecdsa_ctx* ctx, const uint32_t* data, const int* item_limbs, int n_items, uint32_t* digest, size_t count, int mem);
/* `HashCommitment::<Sha256>::create_commitment_with_user_defined_randomness(from_bytes(P.to_bytes(true)), blind)`
 * (gg_2020/party_i.rs:577-580,654-659): blind 8 limbs, commitment 8 limbs.                                           */
int tecdsa_hash_commitment_batch(tecdsa_ctx* ctx, const uint32_t* points, const uint32_t* blind, uint32_t* com, size_t count, int mem);

/* ---- other protocols on the same primitives (SURVEY.md section 8(f) rank 4) -------------------------------------------------
 * Lindell-2017 two-party ECDSA (src/protocols/two_party_ecdsa/lindell_2017/{party_one,party_two}.rs).  Key generation is a
 * composition of calls above (DLogProof, hash commitments, NiCorrectKeyProof, PDL-with-slack, CompositeDLogProof):
 * multi-party-ecdsa_b200/lindell17.py.  Entry points of the signing path, all randomness explicit:
 * l17_eph_create: `party_one::EphKeyGenFirstMsg::create` (party_one.rs:403-433) when the four commitment buffers are NULL,
 *   `party_two::EphKeyGenFirstMsg::create_commitments` (party_two.rs:314-371) when given: public_share = k G, c = k base_point2,
 *   ECDDHProof (a1 16 | a2 16 | z 8, nonce = its sampled s), pk_commitment = commit(compressed public_share; pk_blind),
 *   zk_pok_commitment = commit(H(a1, a2); zk_pok_blind).  secret_share and nonce must be non-zero mod q (Scalar::random()).
 * l17_eph_verify: `party_one::EphKeyGenSecondMsg::verify_commitments_and_dlog_proof` (party_one.rs:436-482) with the
 *   commitment buffers, `party_two::EphKeyGenSecondMsg::verify_and_decommit` (party_two.rs:374-387) without; status
 *   TECDSA_ST_OK / _COMMITMENT / _PROOF.
 * l17_partial_sig: `party_two::PartialSig::compute` (party_two.rs:390-424): n [n_keys][64] (key_idx as in paillier_encrypt),
 *   c_key = encrypted_secret_share [count][128], x2, k2 8 limbs, eph_other_public 16, message 8 (reduced mod q), rho 16
 *   (< q^2), randomness 64 (the r of `Paillier::encrypt`) -> c3 [count][128] = c_key^v * Enc(rho q + k2^-1 m) mod N^2 as ONE
 *   job modulo N^2 per element; status _NOT_INVERTIBLE for k2 = 0 (the reference panics), _INVALID_KEY for a bad point.
 * l17_sign: `party_one::Signature::compute_with_recid` (party_one.rs:519-564; `compute` :486-517 returns the same r, s) under
 *   the Paillier key row `key_row` of an uploaded key set; status as above.
 * l17_verify: `party_one::verify` (party_one.rs:567-592): r must equal the UNREDUCED x coordinate of u1 G + u2 Y and s < q - s;
 *   status TECDSA_ST_OK / _INVALID_SIG.                                                                                      */
int tecdsa_l17_eph_create_batch(tecdsa_ctx* ctx, const uint32_t* secret_share, const uint32_t* nonce, const uint32_t* pk_blind,
                                const uint32_t* zk_pok_blind, uint32_t* public_share, uint32_t* c_point, uint32_t* proof,
                                uint32_t* pk_commitment, uint32_t* zk_pok_commitment, size_t count, int mem);
int tecdsa_l17_eph_verify_batch(tecdsa_ctx* ctx, const uint32_t* public_share, const uint32_t* c_point, const uint32_t* proof,
                                const uint32_t* pk_blind, const uint32_t* zk_pok_blind, const uint32_t* pk_commitment,
                                const uint32_t* zk_pok_commitment, uint8_t* status, size_t count, int mem);
int tecdsa_l17_partial_sig_batch(tecdsa_ctx* ctx, const uint32_t* n, const uint32_t* key_idx, size_t n_keys, const uint32_t* c_key,
                                 const uint32_t* x2, const uint32_t* k2, const uint32_t* eph_other_public, const uint32_t* message,
                                 const uint32_t* rho, const uint32_t* randomness, uint32_t* c3, uint8_t* status, size_t count, int mem);
int tecdsa_l17_sign_batch(tecdsa_ctx* ctx, const tecdsa_keyset* ks, const uint32_t* key_row, const uint32_t* c3, const uint32_t* k1,
                          const uint32_t* eph_other_public, uint32_t* sig_r, uint32_t* sig_s, uint8_t* recid, uint8_t* status,
                          size_t count, int mem);
int tecdsa_l17_verify_batch(tecdsa_ctx* ctx, const uint32_t* sig_r, const uint32_t* sig_s, const uint32_t* pubkey, const uint32_t* message,
                            uint8_t* status, size_t count, int mem);
/* The interactive PDL proof of src/utilities/zk_pdl/mod.rs WITHOUT its `RangeProofNi` (zk-paillier, out of tree, not restated):
 * verifier_message1 (:111-148): a 8 limbs (< q), b 16 (< q^2), randomness 64 (of `Paillier::encrypt(b)`), blindness 8 ->
 *   c_tag [128] = c^a * Enc(b) mod N^2 (one job), c_tag_tag [8] = commit(a + (b << bit_length(a)); blindness), q_tag = a Q + b G;
 * prover_message1 (:191-215): alpha [64] = Dec(c_tag) under key row `key_row`, q_hat = (alpha mod q) G, c_hat = commit(compressed
 *   q_hat; blindness);  prover_message2 (:217-243): status _OK iff a x1 + b == alpha over the integers and c_tag_tag reopens,
 *   else _PDL_VERIFY;  verifier_finalize (:170-187): c_hat reopens and q_hat == q_tag, else _PDL_VERIFY.                        */
int tecdsa_zkpdl_verifier_message1_batch(tecdsa_ctx* ctx, const uint32_t* n, const uint32_t* key_idx, size_t n_keys, const uint32_t* ciphertext,
                                         const uint32_t* Q, const uint32_t* a, const uint32_t* b, const uint32_t* randomness,
                                         const uint32_t* blindness, uint32_t* c_tag, uint32_t* c_tag_tag, uint32_t* q_tag, uint8_t* status,
                                         size_t count, int mem);
int tecdsa_zkpdl_prover_message1_batch(tecdsa_ctx* ctx, const tecdsa_keyset* ks, const uint32_t* key_row, const uint32_t* c_tag,
                                       const uint32_t* blindness, uint32_t* c_hat, uint32_t* q_hat, uint32_t* alpha, uint8_t* status,
                                       size_t count, int mem);
int tecdsa_zkpdl_prover_message2_batch(tecdsa_ctx* ctx, const uint32_t* x1, const uint32_t* alpha, const uint32_t* c_tag_tag, const uint32_t* a,
                                       const uint32_t* b, const uint32_t* blindness, uint8_t* status, size_t count, int mem);
int tecdsa_zkpdl_verifier_finalize_batch(tecdsa_ctx* ctx, const uint32_t* c_hat, const uint32_t* q_hat, const uint32_t* blindness,
                                         const uint32_t* q_tag, uint8_t* status, size_t count, int mem);
/* GG18 signing, the phases GG20 replaced (src/protocols/multi_party_ecdsa/gg_2018/party_i.rs:455-730); phases 1-3 are the MtA
 * calls above with n_st = 0 plus scalar sums.  A batch is `sessions` signing sessions of `parties` signers; element
 * u = session * parties + party, every array element-major, "the other signers" = the other elements of the session.
 * phase4 (:455-485): b_proof_pk [count][parties][16] (entry j = pk of the DLogProof received from signer j; own entry = own
 *   g^gamma), g_gamma 16, blind 8, com 8 per element -> R = delta_inv * sum g_gamma; status _OK / _INVALID_KEY.
 * local_sig (:489-511): s_i = m k_i + r sigma_i.
 * phase5a (:513-558): -> com 8, decom = V 16 | A 16 | B 16, HomoELGamalProof (T 16 | A3 16 | z1 8 | z2 8) for the statement
 *   (G = A, H = R, Y = generator, D = V, E = B), DLogProof of rho (40 limbs); every scalar input non-zero mod q.
 * phase5c (:560-629): checks the OTHER signers' phase-5a messages (commitment, ElGamal proof, DLog proof) -> com2 8,
 *   decom2 = u_i 16 | t_i 16; status _OK / _COMMITMENT (Err(InvalidCom)) / _INVALID_SIG (identity point in a transcript).
 * phase5d (:631-665) over all signers' second messages: status _OK / _COMMITMENT / _INVALID_KEY.
 * output_signature (:666-703) + `verify` (:706-730): every element derives (r, s, recid) of its session; _OK / _INVALID_SIG.      */
int tecdsa_gg18_phase4_batch(tecdsa_ctx* ctx, int parties, const uint32_t* delta_inv, const uint32_t* b_proof_pk, const uint32_t* g_gamma,
                             const uint32_t* blind, const uint32_t* com, uint32_t* R, uint8_t* status, size_t sessions, int mem);
int tecdsa_gg18_local_sig_batch(tecdsa_ctx* ctx, const uint32_t* message, const uint32_t* R, const uint32_t* k_i, const uint32_t* sigma_i,
                                uint32_t* s_i, size_t count, int mem);
int tecdsa_gg18_phase5a_batch(tecdsa_ctx* ctx, const uint32_t* R, const uint32_t* s_i, const uint32_t* l_i, const uint32_t* rho_i,
                              const uint32_t* blind, const uint32_t* heg_s1, const uint32_t* heg_s2, const uint32_t* dlog_nonce,
                              uint32_t* com, uint32_t* decom, uint32_t* heg_proof, uint32_t* dlog_proof, uint8_t* status, size_t count, int mem);
int tecdsa_gg18_phase5c_batch(tecdsa_ctx* ctx, int parties, const uint32_t* R, const uint32_t* y, const uint32_t* message, const uint32_t* rho_i,
                              const uint32_t* l_i, const uint32_t* blind2, const uint32_t* com, const uint32_t* decom, const uint32_t* blind,
                              const uint32_t* heg_proof, const uint32_t* dlog_proof, uint32_t* com2, uint32_t* decom2, uint8_t* status,
                              size_t sessions, int mem);
int tecdsa_gg18_phase5d_batch(tecdsa_ctx* ctx, int parties, const uint32_t* decom2, const uint32_t* blind2, const uint32_t* com2,
                              const uint32_t* decom, uint8_t* status, size_t sessions, int mem);
int tecdsa_gg18_output_signature_batch(tecdsa_ctx* ctx, int parties, const uint32_t* R, const uint32_t* y, const uint32_t* message,
                                       const uint32_t* s_i, uint32_t* sig_r, uint32_t* sig_s, uint8_t* recid, uint8_t* status,
                                       size_t sessions, int mem);

/* ---- L3: the batched GG20 offline-signing stage ----------------------------------------
 * One "unit" = one party's OfflineStage Round0..Round6
 *   (src/protocols/multi_party_ecdsa/gg_2020/state_machine/sign/rounds.rs:68-636,
 *    calling gg_2020/party_i.rs:526-848, utilities/mta/{mod,range_proofs}.rs,
 *    utilities/zk_pdl_with_slack/mod.rs) for keygen parameters t = 1, n = 3 and two signers.
 * A session is two units (2s, 2s+1); both run on the same GPU and exchange their messages in
 * device memory.  The LocalKey material (keygen/rounds.rs:310-322) is uploaded once per key
 * set; per-key constants (N^2, p^2, q^2, the CRT constants of Paillier decrypt) are derived
 * on the device.
 * Accepted keys are those the reference's keygen accepts (gg_2020/party_i.rs:49-50, 287-290):
 * odd p != q, both below 2^1024, with 2^2046 <= N = pq < 2^2048 (so each factor is above
 * 2^1022 and p/q < 4), and 2^2046 <= N_tilde < 2^2048, odd.  Any other row makes
 * tecdsa_keys_upload return TECDSA_E_ARG before anything is allocated.                    */
typedef struct {
    size_t n_keysets;             /* rows below are indexed by keyset*3 + party (party 0..2)      */
    const uint32_t* paillier_p;   /* [rows][32]  DecryptionKey.p  (odd prime, see above)           */
    const uint32_t* paillier_q;   /* [rows][32]  DecryptionKey.q                                   */
    const uint32_t* n_tilde;      /* [rows][64]  DLogStatement.N   (h1_h2_n_tilde_vec)             */
    const uint32_t* h1;           /* [rows][64]  DLogStatement.g                                   */
    const uint32_t* h2;           /* [rows][64]  DLogStatement.ni                                  */
    const uint32_t* x_i;          /* [rows][8]   keys_linear.x_i                                   */
    const uint32_t* pk;           /* [rows][16]  pk_vec[j] = x_j * G, affine x||y                  */
    const uint32_t* y;            /* [n_keysets][16]  y_sum_s                                      */
} tecdsa_keys;
int tecdsa_keys_upload(tecdsa_ctx* ctx, const tecdsa_keys* keys, tecdsa_keyset** out);
int tecdsa_keys_free(tecdsa_ctx* ctx, tecdsa_keyset* ks);
/* copy one derived per-key table back (test access): 0 = N, 1 = N^2, 5 = p^2, 6 = q^2 ... see csrc/gg20_fields.h */
int tecdsa_keys_table(tecdsa_ctx* ctx, const tecdsa_keyset* ks, int table, uint32_t* out_host);

/* Layout (uint32 limb offsets) of one unit's randomness record: every value the reference
 * samples inside OfflineStage, in order of use.  Ranges are the caller's contract and are those
 * of the reference: scalars in [1,q); r_k, beta', r' below the respective Paillier N;
 * alpha < q^3, beta in Z*_N, gamma < q^3 N~, rho < q N~ (utilities/mta/range_proofs.rs:48-51,
 * utilities/zk_pdl_with_slack/mod.rs:73-77).                                                */
enum {
    TECDSA_RND_GAMMA = 0, TECDSA_RND_K = 8, TECDSA_RND_BLIND = 16, TECDSA_RND_RK = 24,
    TECDSA_RND_ALICE = 88, TECDSA_RND_ALICE_STRIDE = 248,       /* x 3 statements                  */
    TECDSA_RND_ALICE_ALPHA = 0, TECDSA_RND_ALICE_BETA = 24, TECDSA_RND_ALICE_GAMMA = 88, TECDSA_RND_ALICE_RHO = 176,
    TECDSA_RND_BETATAG_GAMMA = 832, TECDSA_RND_R_GAMMA = 896, TECDSA_RND_NONCE_GAMMA_B = 960, TECDSA_RND_NONCE_GAMMA_BETA = 968,
    TECDSA_RND_BETATAG_W = 976, TECDSA_RND_R_W = 1040, TECDSA_RND_NONCE_W_B = 1104, TECDSA_RND_NONCE_W_BETA = 1112,
    TECDSA_RND_L = 1120, TECDSA_RND_PED_S1 = 1128, TECDSA_RND_PED_S2 = 1136,
    TECDSA_RND_PDL_ALPHA = 1144, TECDSA_RND_PDL_BETA = 1168, TECDSA_RND_PDL_RHO = 1232, TECDSA_RND_PDL_GAMMA = 1304,
    TECDSA_RND_HEG_S1 = 1392, TECDSA_RND_HEG_S2 = 1400,
    TECDSA_RND_LIMBS = 1408
};

/* sessions[s] = {keyset, party of signer position 0, party of signer position 1} (parties 0..2,
 * i.e. keygen index - 1; `s_l` of OfflineStage::new, sign.rs:78).  rnd = [2*n_sessions][TECDSA_RND_LIMBS].
 * Outputs per unit (any may be NULL except status): status byte (TECDSA_ST_*; first failing check
 * of that party), R (affine x||y, 16 limbs), sigma_i (8 limbs), t_vec (2 x 16 limbs) — the fields
 * of CompletedOfflineStage (sign/rounds.rs:647-654) — and a SHA-256 digest (8 limbs) over every
 * message the unit emitted in a fixed-width canonical encoding (the result record that the
 * multi-GPU gather collects and that the parity tests compare with the oracle).
 * Declared work-saving identities, all value-preserving: the three AliceProof::verify of a peer's
 * MessageA are evaluated once for the two MessageB::b calls (mta/mod.rs:123-131); (N+1)^x mod N^2 is
 * evaluated as 1 + xN; (z^-1)^e as (z^e)^-1; Paillier decrypt's per-key constants are cached.   */
int tecdsa_gg20_offline_batch(tecdsa_ctx* ctx, const tecdsa_keyset* ks, const uint32_t* sessions, size_t n_sessions,
                              const uint32_t* rnd, uint8_t* status, uint32_t* R, uint32_t* sigma, uint32_t* t_vec,
                              uint32_t* digest, int mem);
/* ---- result records, their multi-GPU gather, and the end-to-end call ---------------------------------------------------
 * One 256-byte record per unit (SURVEY.md section 8e) = the fields of CompletedOfflineStage (sign/rounds.rs:647-654) in the
 * reference's byte encodings: status byte, R and t_vec as `Point::to_bytes(true)` (33 bytes), sigma_i and k_i
 * (`sign_keys.k_i`) as 32-byte big-endian scalars, and the 32-byte transcript digest; the rest is zero.                  */
enum {
    TECDSA_REC_BYTES = 256, TECDSA_REC_STATUS = 0, TECDSA_REC_R = 1, TECDSA_REC_SIGMA = 34, TECDSA_REC_K = 66,
    TECDSA_REC_T0 = 98, TECDSA_REC_T1 = 131, TECDSA_REC_DIGEST = 164
};
/* records[u] from the per-unit outputs of tecdsa_gg20_offline_batch and the batch's randomness records (k_i); DEVICE pointers. */
int tecdsa_gg20_pack_records(tecdsa_ctx* ctx, const uint8_t* status, const uint32_t* R, const uint32_t* sigma, const uint32_t* t_vec,
                             const uint32_t* digest, const uint32_t* rnd, size_t n_units, uint8_t* records);
/* The single collective of the path: all_records[rank][n_units][256] on every rank = ncclAllGather of each rank's
 * records[n_units][256] on the context stream (DEVICE pointers; `nccl_comm` is an ncclComm_t; NULL = one rank, a copy).
 * NCCL is bound at run time to the libnccl.so.2 already loaded in the process (no link-time dependency).                 */
int tecdsa_gather_results(tecdsa_ctx* ctx, void* nccl_comm, const uint8_t* records, size_t n_units, uint8_t* all_records);
/* Communicator plumbing for callers that do not already hold an ncclComm_t: rank 0 draws an id (`ncclGetUniqueId`) and
 * distributes its 128 bytes out of band; every rank then creates its communicator for the context's device.             */
enum { TECDSA_NCCL_ID_BYTES = 128 };
int tecdsa_nccl_unique_id(uint8_t id[TECDSA_NCCL_ID_BYTES]);
int tecdsa_nccl_comm_create(tecdsa_ctx* ctx, const uint8_t id[TECDSA_NCCL_ID_BYTES], int nranks, int rank, void** nccl_comm);
int tecdsa_nccl_comm_destroy(void* nccl_comm);
/* End to end: sessions / rnd as for tecdsa_gg20_offline_batch; H2D of the inputs -> Round0..6 -> pack -> gather -> D2H, all on
 * the context stream.  all_records = [nranks][2*n_sessions][256] (nranks = 1 when nccl_comm == NULL); with TECDSA_HOST the
 * call returns after the records have landed in host memory.                                                            */
int tecdsa_gg20_offline_records(tecdsa_ctx* ctx, const tecdsa_keyset* ks, void* nccl_comm, const uint32_t* sessions, size_t n_sessions,
                                const uint32_t* rnd, uint8_t* all_records, int mem);
/* ---- online step (gg_2020/party_i.rs:850-936) for a batch of completed two-signer sessions ------------------------------
 * message = [n_sessions][8] (the BigInt being signed, reduced mod q like `Scalar::from`), R / sigma / k = per-unit outputs of
 * the offline stage ([2n][16], [2n][8], [2n][8]).  s_i (optional, [2n][8]) = `phase7_local_sig`: m k_i + r sigma_i;
 * (sig_r, sig_s, recid) = `output_signature` over both signers' s_i (low-s normalised); status = TECDSA_ST_OK or
 * TECDSA_ST_INVALID_SIG from the in-tree `verify` against the key set's y (Error::InvalidSig, party_i.rs:908,934).       */
int tecdsa_gg20_sign_batch(tecdsa_ctx* ctx, const tecdsa_keyset* ks, const uint32_t* sessions, size_t n_sessions, const uint32_t* message,
                           const uint32_t* R, const uint32_t* sigma, const uint32_t* k, uint32_t* s_i, uint32_t* sig_r, uint32_t* sig_s,
                           uint8_t* recid, uint8_t* status, int mem);
/* 32x32+64 multiply-accumulates executed by the big-integer kernels of this context since creation / the last reset:
 * counted by the kernels themselves (one atomic add per job, from the loop trip counts of the products it ran) — the
 * "ops actually executed" figure of SURVEY.md section 8(d).  EC / hashing glue and the shift-subtract inversions are not
 * multiply-accumulate work and are not counted.                                                                          */
int tecdsa_ctx_work(tecdsa_ctx* ctx, uint64_t* mac32, int reset);
/* Per-launch profiling: while enabled, every kernel launch of this context is bracketed by CUDA events on the context stream
 * and the executed-work counter is snapshotted after it (batches then run on the one stream, without the two-stream split).
 * profile_read waits for the stream and returns up to `cap` launches in launch order; *n = how many were recorded.          */
typedef struct { char kernel[48]; float ms; uint64_t mac32; } tecdsa_launch_info;
int tecdsa_ctx_profile(tecdsa_ctx* ctx, int enable);
int tecdsa_ctx_profile_read(tecdsa_ctx* ctx, tecdsa_launch_info* out, size_t cap, size_t* n);
/* test access: copy one named per-unit field of the last batch (names in csrc/gg20_fields.h) */
int tecdsa_gg20_debug_field(tecdsa_ctx* ctx, const char* name, uint32_t* out_host, size_t* limbs_per_unit);

/* Saturation micro-benchmarks of the integer multiply-add pipe, 32x32+64 MACs per second on this device — the roofline
 * denominators of every kernel of this library (SURVEY.md section 8(d)).  imad_peak: carry-free IMAD.WIDE.U32 on 16 independent
 * accumulators per thread, every product with its own operand pair; imad_peak_chained: IMAD.WIDE.U32.X in the carry chains of
 * the Montgomery rows (two accumulator sets per thread).  Both at full occupancy; tools/sass_mix.py prints their SASS mix.      */
int tecdsa_imad_peak(tecdsa_ctx* ctx, double* mac32_per_s, float* ms);
int tecdsa_imad_peak_chained(tecdsa_ctx* ctx, double* mac32_per_s, float* ms);

#ifdef __cplusplus
}
#endif
#endif
