// L0 / L1 / L2 batch entry points (include/tecdsa_b200.h): the scalar calls of curv-kzen
// `BigInt`, kzen-paillier `Paillier::*` and the in-tree MtA range proof, batched.  They are thin
// compositions of the same job-list kernels and glue device functions the L3 offline-stage
// driver uses (jobs.cuh, modinv.cuh, gg20_glue.cuh); results are canonical residues /
// proof bytes identical to the L3 path and to the oracle.
#include "stage.cuh"
#include "l12_steps.h"

using namespace tecdsa;

namespace {

// ---- glue kernels of the stand-alone entry points ----------------------------------------------
// out[i] (128 limbs) = 1 + m[i] * N[row]      (the (1 + m n) factor of Paillier encrypt)
__global__ void k_lin(uint32_t* out, const uint32_t* m, int m_limbs, const uint32_t* n_tab, const uint32_t* rows, int count) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    uint32_t one = 1;
    st::mul_add(out + (size_t)i * 128, 128, m + (size_t)i * m_limbs, m_limbs, n_tab + (size_t)(rows ? rows[i] : i) * 64, 64, &one, 1);
}
__global__ void k_secp_mul(uint32_t* out, const uint32_t* pts, const uint32_t* scalars, int count) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    U256 k = sc_from_limbs(scalars + (size_t)i * 8, 8);
    Affine r;
    if (!pts) r = mul_G(k);                                    // generator: fixed-base tables
    else {
        Affine P = affine_load(pts + (size_t)i * 16);
        if (!P.inf && !on_curve(P)) { r.inf = true; r.x = u256_zero(); r.y = u256_zero(); }
        else r = pt_mul(P, k);
    }
    affine_store(out + (size_t)i * 16, r);
}
// AliceProof::generate middle: e, s1, s2   (range_proofs.rs:174-182, 87-88)
__global__ void k_alice_mid(Arena A, const uint32_t* ek_rows, const uint32_t* cipher, const uint32_t* z, const uint32_t* u, const uint32_t* w,
                            const uint32_t* a, const uint32_t* alpha, const uint32_t* gamma, const uint32_t* rho, uint32_t* e, uint32_t* s1,
                            uint32_t* s2, int count) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    uint32_t* ei = e + (size_t)i * 8;
    alice_hash(ei, A.k(KT_N, ek_rows[i]), cipher + (size_t)i * 128, z + (size_t)i * 64, u + (size_t)i * 128, w + (size_t)i * 64);
    st::mul_add(s1 + (size_t)i * 28, 28, ei, 8, a + (size_t)i * 8, 8, alpha + (size_t)i * 24, 24);
    st::mul_add(s2 + (size_t)i * 92, 92, ei, 8, rho + (size_t)i * 72, 72, gamma + (size_t)i * 88, 88);
}
// AliceProof::verify prologue: range check + gs1 = s1 N + 1   (range_proofs.rs:118,134)
__global__ void k_alice_vpre(Arena A, const uint32_t* ek_rows, const uint32_t* s1, uint32_t* gs1, uint8_t* range_bad, int count) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    const uint32_t* s = s1 + (size_t)i * 28;
    range_bad[i] = st::cmp2(s, 28, Q3_LIMBS, 24) > 0;
    uint32_t one = 1;
    st::mul_add(gs1 + (size_t)i * 128, 128, s, 28, A.k(KT_N, ek_rows[i]), 64, &one, 1);
}
// AliceProof::verify epilogue: recompute e and compare   (range_proofs.rs:143-153)
__global__ void k_alice_vpost(Arena A, const uint32_t* ek_rows, const uint32_t* cipher, const uint32_t* z, const uint32_t* u, const uint32_t* w,
                              const uint32_t* e, const uint8_t* range_bad, const uint8_t* okz, const uint8_t* okc, uint32_t* e_scratch,
                              uint8_t* status, int count) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    uint8_t st_ = TECDSA_ST_OK;
    if (range_bad[i]) st_ = TECDSA_ST_RANGE;
    else if (!okz[i] || !okc[i]) st_ = TECDSA_ST_NOT_INVERTIBLE;
    else {
        uint32_t* ei = e_scratch + (size_t)i * 8;
        alice_hash(ei, A.k(KT_N, ek_rows[i]), cipher + (size_t)i * 128, z + (size_t)i * 64, u + (size_t)i * 128, w + (size_t)i * 64);
        if (st::cmp(ei, e + (size_t)i * 8, 8) != 0) st_ = TECDSA_ST_HASH_MISMATCH;
    }
    status[i] = st_;
}


// ---- PDL with slack (utilities/zk_pdl_with_slack/mod.rs:68-179) -------------------------------------
// prove, first part: u1 = G * alpha, lin = 1 + alpha N
__global__ void k_pdl_pre(Arena A, const uint32_t* ek_rows, const uint32_t* Gp, const uint32_t* alpha, uint32_t* u1, uint32_t* lin, int count) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    affine_store(u1 + (size_t)i * 16, pt_mul(affine_load(Gp + (size_t)i * 16), sc_from_limbs(alpha + (size_t)i * 24, 24)));
    uint32_t one = 1;
    st::mul_add(lin + (size_t)i * 128, 128, alpha + (size_t)i * 24, 24, A.k(KT_N, ek_rows[i]), 64, &one, 1);
}
// e, s1 = e x + alpha, s3 = e rho + gamma  (:102-114)
__global__ void k_pdl_mid(const uint32_t* Gp, const uint32_t* Qp, const uint32_t* cipher, const uint32_t* z, const uint32_t* u1, const uint32_t* u2,
                          const uint32_t* u3, const uint32_t* x, const uint32_t* alpha, const uint32_t* rho, const uint32_t* gamma,
                          uint32_t* e, uint32_t* s1, uint32_t* s3, int count) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    uint32_t* ei = e + (size_t)i * 8;
    pdl_hash(ei, affine_load(Gp + (size_t)i * 16), affine_load(Qp + (size_t)i * 16), cipher + (size_t)i * 128, z + (size_t)i * 64,
             affine_load(u1 + (size_t)i * 16), u2 + (size_t)i * 128, u3 + (size_t)i * 64);
    st::mul_add(s1 + (size_t)i * 28, 28, ei, 8, x + (size_t)i * 8, 8, alpha + (size_t)i * 24, 24);
    st::mul_add(s3 + (size_t)i * 92, 92, ei, 8, rho + (size_t)i * 72, 72, gamma + (size_t)i * 88, 88);
}
// verify prologue: e (into scratch) and lin = 1 + s1 N  (:128-150)
__global__ void k_pdl_vpre(Arena A, const uint32_t* ek_rows, const uint32_t* Gp, const uint32_t* Qp, const uint32_t* cipher, const uint32_t* z,
                           const uint32_t* u1, const uint32_t* u2, const uint32_t* u3, const uint32_t* s1, uint32_t* e, uint32_t* lin, int count) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    pdl_hash(e + (size_t)i * 8, affine_load(Gp + (size_t)i * 16), affine_load(Qp + (size_t)i * 16), cipher + (size_t)i * 128, z + (size_t)i * 64,
             affine_load(u1 + (size_t)i * 16), u2 + (size_t)i * 128, u3 + (size_t)i * 64);
    uint32_t one = 1;
    st::mul_add(lin + (size_t)i * 128, 128, s1 + (size_t)i * 28, 28, A.k(KT_N, ek_rows[i]), 64, &one, 1);
}
// verify epilogue: u1 == G s1 + Q (-e), u2 == u2', u3 == u3'  (:138-178)
__global__ void k_pdl_vpost(const uint32_t* Gp, const uint32_t* Qp, const uint32_t* u1, const uint32_t* u2, const uint32_t* u3, const uint32_t* s1,
                            const uint32_t* e, const uint32_t* u2t, const uint32_t* u3t, const uint8_t* okz, const uint8_t* okc, uint8_t* status, int count) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    Affine G_ = affine_load(Gp + (size_t)i * 16), Q_ = affine_load(Qp + (size_t)i * 16), U1 = affine_load(u1 + (size_t)i * 16);
    bool ok = okz[i] && okc[i] && on_curve(G_) && on_curve(Q_) && on_curve(U1);
    if (ok) {
        Affine t = lin2(G_, sc_from_limbs(s1 + (size_t)i * 28, 28), Q_, sc_neg(sc_from_limbs(e + (size_t)i * 8, 8)));
        ok = affine_eq(t, U1) && st::cmp(u2t + (size_t)i * 128, u2 + (size_t)i * 128, 128) == 0 &&
             st::cmp(u3t + (size_t)i * 64, u3 + (size_t)i * 64, 64) == 0;
    }
    status[i] = ok ? TECDSA_ST_OK : TECDSA_ST_PDL_VERIFY;
}

// ---- Bob's MtA / MtAwc range proof (utilities/mta/range_proofs.rs:214-535) ----------------------------
// lin = (x mod N) * N + 1 for x of xl limbs (x may exceed N: gamma < q^2 N, t1 = e beta' + gamma)
__global__ void k_lin_wide(Arena A, const uint32_t* ek_rows, const uint32_t* x, int xl, uint32_t* lin, int count) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    const uint32_t* N = A.k(KT_N, ek_rows[i]);
    uint32_t red[64], one = 1;
    st::mod_slow(red, x + (size_t)i * xl, xl, N, 64);
    st::mul_add(lin + (size_t)i * 128, 128, red, 64, N, 64, &one, 1);
}
__device__ void bob_hash(uint32_t* e8, const uint32_t* N, const uint32_t* a_enc, const uint32_t* mta, const uint32_t* z, const uint32_t* zp,
                         const uint32_t* t, const uint32_t* v, const uint32_t* w, const Affine* X, const Affine* U) {
    Sha256 h; h.init();
    h.put_bigint(N, 64);
    uint32_t n1[65];
    uint64_t cy = 1;
    for (int i = 0; i < 64; i++) { cy += N[i]; n1[i] = (uint32_t)cy; cy >>= 32; }
    n1[64] = (uint32_t)cy;
    h.put_bigint(n1, 65);
    h.put_bigint(a_enc, 128); h.put_bigint(mta, 128); h.put_bigint(z, 64); h.put_bigint(zp, 64); h.put_bigint(t, 64);
    h.put_bigint(v, 128); h.put_bigint(w, 64);
    if (X) { h.put_bigint(X->x.v, 8); h.put_bigint(X->y.v, 8); h.put_bigint(U->x.v, 8); h.put_bigint(U->y.v, 8); }   // coordinates as BigInt (:386-395)
    h.finish(e8);
}
// generate: e and the five plain-integer responses (:433-470, 289-296); with `check` also X = G b, u = G alpha
__global__ void k_bob_mid(Arena A, const uint32_t* ek_rows, int check, const uint32_t* a_enc, const uint32_t* mta, const uint32_t* z, const uint32_t* zp,
                          const uint32_t* t, const uint32_t* v, const uint32_t* w, const uint32_t* b, const uint32_t* beta_prim, const uint32_t* alpha,
                          const uint32_t* gamma, const uint32_t* ro, const uint32_t* ro_prim, const uint32_t* sigma, const uint32_t* tau,
                          uint32_t* e, uint32_t* s1, uint32_t* s2, uint32_t* t1, uint32_t* t2, uint32_t* u_out, int count) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    uint32_t* ei = e + (size_t)i * 8;
    Affine X, U;
    if (check) {
        X = mul_G(sc_from_limbs(b + (size_t)i * 8, 8));
        U = mul_G(sc_from_limbs(alpha + (size_t)i * 24, 24));
        affine_store(u_out + (size_t)i * 16, U);
    }
    bob_hash(ei, A.k(KT_N, ek_rows[i]), a_enc + (size_t)i * 128, mta + (size_t)i * 128, z + (size_t)i * 64, zp + (size_t)i * 64, t + (size_t)i * 64,
             v + (size_t)i * 128, w + (size_t)i * 64, check ? &X : nullptr, check ? &U : nullptr);
    st::mul_add(s1 + (size_t)i * 28, 28, ei, 8, b + (size_t)i * 8, 8, alpha + (size_t)i * 24, 24);
    st::mul_add(s2 + (size_t)i * 92, 92, ei, 8, ro + (size_t)i * 72, 72, ro_prim + (size_t)i * 88, 88);
    st::mul_add(t1 + (size_t)i * 84, 84, ei, 8, beta_prim + (size_t)i * 64, 64, gamma + (size_t)i * 80, 80);
    st::mul_add(t2 + (size_t)i * 92, 92, ei, 8, sigma + (size_t)i * 72, 72, tau + (size_t)i * 88, 88);
}
__global__ void k_bob_vpre(const uint32_t* s1, uint8_t* range_bad, int count) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    range_bad[i] = st::cmp2(s1 + (size_t)i * 28, 28, Q3_LIMBS, 24) > 0;
}
// verify epilogue (:374-410) and, for BobProofExt, G s1 == X e + u (:522-531)
__global__ void k_bob_vpost(Arena A, const uint32_t* ek_rows, const uint32_t* a_enc, const uint32_t* mta, const uint32_t* z, const uint32_t* zp,
                            const uint32_t* t, const uint32_t* v, const uint32_t* w, const uint32_t* e, const uint32_t* s1, const uint32_t* Xp,
                            const uint32_t* Up, const uint8_t* range_bad, const uint8_t* ok1, const uint8_t* ok2, const uint8_t* ok3,
                            uint32_t* e_scratch, uint8_t* status, int count) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    uint8_t st_ = TECDSA_ST_OK;
    if (range_bad[i]) st_ = TECDSA_ST_RANGE;
    else if (!ok1[i] || !ok2[i] || !ok3[i]) st_ = TECDSA_ST_NOT_INVERTIBLE;
    else {
        Affine X, U;
        if (Xp) { X = affine_load(Xp + (size_t)i * 16); U = affine_load(Up + (size_t)i * 16); }
        uint32_t* ei = e_scratch + (size_t)i * 8;
        bob_hash(ei, A.k(KT_N, ek_rows[i]), a_enc + (size_t)i * 128, mta + (size_t)i * 128, z + (size_t)i * 64, zp + (size_t)i * 64,
                 t + (size_t)i * 64, v + (size_t)i * 128, w + (size_t)i * 64, Xp ? &X : nullptr, Xp ? &U : nullptr);
        if (st::cmp(ei, e + (size_t)i * 8, 8) != 0) st_ = TECDSA_ST_HASH_MISMATCH;
        else if (Xp) {
            if (X.inf || U.inf || !on_curve(X) || !on_curve(U)) st_ = TECDSA_ST_PROOF;
            else {
                Affine x1 = mul_G(sc_from_limbs(s1 + (size_t)i * 28, 28));
                Affine x2 = jac_to_affine(jac_add(jac_mul(jac_from_affine(X), sc_from_limbs(e + (size_t)i * 8, 8)), jac_from_affine(U)));
                if (!affine_eq(x1, x2)) st_ = TECDSA_ST_PROOF;
            }
        }
    }
    status[i] = st_;
}


// ---- curv sigma proofs and hashes as stand-alone batches ------------------------------------------------
__global__ void k_dlog_prove(uint32_t* out40, const uint32_t* sk, const uint32_t* nonce, int count) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    dlog_prove(out40 + (size_t)i * 40, sc_from_limbs(sk + (size_t)i * 8, 8), sc_from_limbs(nonce + (size_t)i * 8, 8));
}
__global__ void k_dlog_verify(const uint32_t* in40, uint8_t* status, int count) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    status[i] = dlog_verify(in40 + (size_t)i * 40) ? TECDSA_ST_OK : TECDSA_ST_PROOF;
}
// PedersenProof::prove [R]: com = m G + r H; a1 = s1 G; a2 = s2 H; e = H(G,H,com,a1,a2); z1 = s1 + e m; z2 = s2 + e r
__global__ void k_pedersen_prove(uint32_t* com16, uint32_t* ped64, const uint32_t* m, const uint32_t* r, const uint32_t* s1, const uint32_t* s2, int count) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    const U256 mm = sc_from_limbs(m + (size_t)i * 8, 8), rr = sc_from_limbs(r + (size_t)i * 8, 8);
    const U256 a = sc_from_limbs(s1 + (size_t)i * 8, 8), b = sc_from_limbs(s2 + (size_t)i * 8, 8);
    Affine pts[5];
    pts[0] = affine_G(); pts[1] = affine_H(); pts[2] = lin_GH(mm, rr); pts[3] = mul_G(a); pts[4] = mul_H(b);
    U256 e = hash_points_scalar(pts, 5);
    uint32_t* ped = ped64 + (size_t)i * 64;
    for (int j = 56; j < 64; j++) ped[j] = 0;
    affine_store(com16 + (size_t)i * 16, pts[2]);
    u256_store(ped, e); affine_store(ped + 8, pts[3]); affine_store(ped + 24, pts[4]);
    u256_store(ped + 40, sc_add(a, sc_mul(e, mm))); u256_store(ped + 48, sc_add(b, sc_mul(e, rr)));
}
__global__ void k_pedersen_verify(const uint32_t* com16, const uint32_t* ped64, uint8_t* status, int count) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    status[i] = pedersen_verify(ped64 + (size_t)i * 64, affine_load(com16 + (size_t)i * 16)) ? TECDSA_ST_OK : TECDSA_ST_PROOF;
}
// HomoELGamalProof::prove [R] for the statement (G, H = base_point2, Y = generator, D, E), witness (x, r)
__global__ void k_heg_prove(uint32_t* heg48, const uint32_t* G16, const uint32_t* D16, const uint32_t* E16, const uint32_t* x, const uint32_t* r,
                            const uint32_t* s1, const uint32_t* s2, int count) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    const U256 xx = sc_from_limbs(x + (size_t)i * 8, 8), rr = sc_from_limbs(r + (size_t)i * 8, 8);
    const U256 a = sc_from_limbs(s1 + (size_t)i * 8, 8), b = sc_from_limbs(s2 + (size_t)i * 8, 8);
    Affine Gp = affine_load(G16 + (size_t)i * 16);
    Affine T = lin_GH(b, a);                       // H*s1 + Y*s2
    Affine A3 = pt_mul(Gp, b);
    U256 e = heg_hash(T, A3, Gp, affine_load(D16 + (size_t)i * 16), affine_load(E16 + (size_t)i * 16));
    uint32_t* heg = heg48 + (size_t)i * 48;
    affine_store(heg, T); affine_store(heg + 16, A3);
    u256_store(heg + 32, u256_is_zero(xx) ? a : sc_add(a, sc_mul(xx, e)));
    u256_store(heg + 40, sc_add(b, sc_mul(rr, e)));
}
__global__ void k_heg_verify(const uint32_t* heg48, const uint32_t* G16, const uint32_t* D16, const uint32_t* E16, uint8_t* status, int count) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    Affine Gp = affine_load(G16 + (size_t)i * 16);
    bool ok = !Gp.inf && on_curve(Gp) && heg_verify(heg48 + (size_t)i * 48, Gp, affine_load(D16 + (size_t)i * 16), affine_load(E16 + (size_t)i * 16));
    status[i] = ok ? TECDSA_ST_OK : TECDSA_ST_PROOF;
}
// `Sha256::new().chain_bigint(x_0)...chain_bigint(x_{k-1}).result_bigint()`: item j of element i has limbs[j] limbs at
// data + i*stride + offset_j (offsets are the running sum of limbs)
__global__ void k_sha256_bigints(const uint32_t* data, int stride, const int* limbs, int n_items, uint32_t* out8, int count) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    Sha256 h; h.init();
    const uint32_t* p = data + (size_t)i * stride;
    for (int j = 0; j < n_items; j++) { h.put_bigint(p, limbs[j]); p += limbs[j]; }
    h.finish(out8 + (size_t)i * 8);
}
// HashCommitment::create_commitment_with_user_defined_randomness(from_bytes(compress(P)), blind)
__global__ void k_hash_commit(const uint32_t* P16, const uint32_t* blind8, uint32_t* out8, int count) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    hash_commit_point(out8 + (size_t)i * 8, affine_load(P16 + (size_t)i * 16), blind8 + (size_t)i * 8);
}


// ---- MtA messages (utilities/mta/mod.rs:52-179) --------------------------------------------------------
// replicate per-instance rows for a flat (instance, statement) proof batch: dst[i*n_st + x] = src[i]
__global__ void k_expand(uint32_t* dst, const uint32_t* src, int limbs, int n_st, int count) {
    int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= count * n_st) return;
    const uint32_t* p = src + (size_t)(t / n_st) * limbs;
    uint32_t* d = dst + (size_t)t * limbs;
    for (int j = 0; j < limbs; j++) d[j] = p[j];
}
// MessageB::b tail: any rejected proof -> InvalidKey; beta = -beta' mod q; the two DLogProofs (mod.rs:123-148)
__global__ void k_mta_b_post(const uint8_t* proof_status, int n_st, const uint32_t* b, const uint32_t* beta_tag, const uint32_t* nonce_b,
                             const uint32_t* nonce_beta, uint32_t* beta_out, uint32_t* b_proof, uint32_t* bt_proof, uint8_t* status, int count) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    bool ok = true;
    for (int x = 0; x < n_st; x++) ok = ok && proof_status[(size_t)i * n_st + x] == TECDSA_ST_OK;
    status[i] = ok ? TECDSA_ST_OK : TECDSA_ST_INVALID_KEY;
    U256 bt = sc_from_limbs(beta_tag + (size_t)i * 64, 64);
    u256_store(beta_out + (size_t)i * 8, sc_neg(bt));
    dlog_prove(b_proof + (size_t)i * 40, sc_from_limbs(b + (size_t)i * 8, 8), sc_from_limbs(nonce_b + (size_t)i * 8, 8));
    dlog_prove(bt_proof + (size_t)i * 40, bt, sc_from_limbs(nonce_beta + (size_t)i * 8, 8));
}
// MessageB::verify_proofs_get_alpha tail (mod.rs:165-178)
__global__ void k_mta_alpha(Arena A, const uint32_t* rows, const uint32_t* dp, const uint32_t* dq, const uint32_t* a, const uint32_t* b_proof,
                            const uint32_t* bt_proof, uint32_t* plain, uint32_t* alpha_out, uint8_t* status, int count) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    uint32_t* pl = plain + (size_t)i * 64;
    decrypt_finish(pl, A, rows[i], dp + (size_t)i * 64, dq + (size_t)i * 64);
    U256 alpha = sc_from_limbs(pl, 64);
    u256_store(alpha_out + (size_t)i * 8, alpha);
    const uint32_t *bp = b_proof + (size_t)i * 40, *btp = bt_proof + (size_t)i * 40;
    Affine g_alpha = mul_G(alpha);
    Affine ba_btag = jac_to_affine(jac_add(jac_mul(jac_from_affine(affine_load(bp)), sc_from_limbs(a + (size_t)i * 8, 8)), jac_from_affine(affine_load(btp))));
    const bool v1 = dlog_verify(bp), v2 = dlog_verify(btp);
    status[i] = (v1 && v2 && affine_eq(ba_btag, g_alpha)) ? TECDSA_ST_OK : TECDSA_ST_INVALID_KEY;
}

}  // namespace

__global__ void k_decrypt_finish(Arena A, uint32_t* out, const uint32_t* dp, const uint32_t* dq, const uint32_t* rows, int count) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    decrypt_finish(out + (size_t)i * 64, A, rows[i], dp + (size_t)i * 64, dq + (size_t)i * 64);
}

int tecdsa_internal_fb_points_set_l12(const uint32_t* table) {
    CK(cudaMemcpyToSymbol(secp::g_fb_points, &table, sizeof(table)));
    return 0;
}


// ------------------------------------------------------------------------------------------ L0
extern "C" int tecdsa_modmul_batch(tecdsa_ctx* c, int mod_bits, const uint32_t* a, const uint32_t* b, const uint32_t* modulus,
                                   const uint32_t* mod_idx, size_t n_mod, uint32_t* out, size_t count, int mem) {
    if (!c || !a || !b || !modulus || !out) return tecdsa_fail(TECDSA_E_ARG, "modmul: null argument");
    if (check_bits(mod_bits)) return TECDSA_E_UNSUPPORTED;
    STAGE_PROLOGUE("modmul", count);
    const int K = mod_bits / 32;
    const uint32_t *da = S.in(a, count * K), *db = S.in(b, count * K), *dm = S.in(modulus, (mod_idx ? n_mod : count) * K), *di = S.in(mod_idx, count);
    uint32_t* dout = S.out(out, count * K);
    if (S.err) return S.err;
    Launches L;
    ExpLaunch& l = K == 64 ? L.e64 : L.e128;
    add_exp(l, K, (int)count, di ? tab(dm, di, K) : arr(dm, K), 0, NONE, NONE, 0, NONE, NONE, 0, 2, arr(da, K), arr(db, K), dout, K);
    RUN(run(c, l, K));
    return S.finish();
}

extern "C" int tecdsa_modinv_batch(tecdsa_ctx* c, int mod_bits, const uint32_t* a, const uint32_t* modulus, const uint32_t* mod_idx,
                                   size_t n_mod, uint32_t* out, uint8_t* ok, size_t count, int mem) {
    if (!c || !a || !modulus || !out || !ok) return tecdsa_fail(TECDSA_E_ARG, "modinv: null argument");
    if (check_bits(mod_bits)) return TECDSA_E_UNSUPPORTED;
    STAGE_PROLOGUE("modinv", count);
    const int K = mod_bits / 32;
    const uint32_t *da = S.in(a, count * K), *dm = S.in(modulus, (mod_idx ? n_mod : count) * K), *di = S.in(mod_idx, count);
    uint32_t* dout = S.out(out, count * K);
    uint8_t* dok = S.out(ok, count);
    if (S.err) return S.err;
    Launches L;
    InvLaunch& l = K == 64 ? L.i64 : L.i128;
    add_inv(l, K, (int)count, di ? tab(dm, di, K) : arr(dm, K), arr(da, K), dout, dok);
    RUN(run(c, l, K));
    return S.finish();
}

extern "C" int tecdsa_secp_mul_batch(tecdsa_ctx* c, const uint32_t* points, const uint32_t* scalars, uint32_t* out, size_t count, int mem) {
    if (!c || !scalars || !out) return tecdsa_fail(TECDSA_E_ARG, "secp_mul: null argument");
    STAGE_PROLOGUE("secp_mul", count);
    const uint32_t *dp = S.in(points, count * 16), *dk = S.in(scalars, count * 8);
    uint32_t* dout = S.out(out, count * 16);
    if (S.err) return S.err;
    RUN(secp_mul_step(c, (int)count, dp, dk, dout));
    return S.finish();
}
// out = k P (k G for pts == NULL) on device-resident arrays
int tecdsa::secp_mul_step(tecdsa_ctx* c, int n, const uint32_t* pts, const uint32_t* scalars, uint32_t* out) {
    k_secp_mul<<<grid_for((size_t)n), 64, 0, c->stream>>>(out, pts, scalars, n);
    KCHECK();
    return 0;
}

// ------------------------------------------------------------------------------------------ L1: Paillier
extern "C" int tecdsa_paillier_encrypt_batch(tecdsa_ctx* c, const uint32_t* n, const uint32_t* key_idx, size_t n_keys, const uint32_t* m,
                                             const uint32_t* r, uint32_t* c_out, size_t count, int mem) {
    if (!c || !n || !m || !r || !c_out) return tecdsa_fail(TECDSA_E_ARG, "paillier_encrypt: null argument");
    STAGE_PROLOGUE("paillier_encrypt", count);
    const uint32_t *dm = S.in(m, count * 64), *dr = S.in(r, count * 64);
    uint32_t* dc = S.out(c_out, count * 128);
    uint32_t* lin = S.tmp<uint32_t>(count * 128);
    if (S.err) return S.err;
    Operand N, ND;
    RUN(stage_caller_key(S, n, key_idx, n_keys, count, N, ND));
    k_lin<<<grid_for(count), 64, 0, c->stream>>>(lin, dm, 64, N.ptr, N.idx, (int)count);
    KCHECK();
    Launches L;
    add_nn(L.e128, (int)count, N, ND, 1, arr(dr, 64), N, 64, NONE, NONE, 0, 1, arr(lin, 128), NONE, dc, 128);     // (1 + m n) * r^n mod n^2
    RUN(run_nn(c, L.e128));
    return S.finish();
}

extern "C" int tecdsa_paillier_mul_batch(tecdsa_ctx* c, const uint32_t* n, const uint32_t* key_idx, size_t n_keys, const uint32_t* ct,
                                         const uint32_t* k, int k_limbs, uint32_t* c_out, size_t count, int mem) {
    if (!c || !n || !ct || !k || !c_out || k_limbs <= 0 || k_limbs > 64) return tecdsa_fail(TECDSA_E_ARG, "paillier_mul: bad argument");
    STAGE_PROLOGUE("paillier_mul", count);
    const uint32_t *dct = S.in(ct, count * 128), *dk = S.in(k, count * (size_t)k_limbs);
    uint32_t* dc = S.out(c_out, count * 128);
    if (S.err) return S.err;
    Operand N, ND;
    RUN(stage_caller_key(S, n, key_idx, n_keys, count, N, ND));
    Launches L;
    add_nn(L.e128, (int)count, N, ND, 1, arr(dct, 128), arr(dk, k_limbs), k_limbs, NONE, NONE, 0, 0, NONE, NONE, dc, 128);
    RUN(run_nn(c, L.e128));
    return S.finish();
}

extern "C" int tecdsa_paillier_add_batch(tecdsa_ctx* c, const uint32_t* n, const uint32_t* key_idx, size_t n_keys, const uint32_t* c1,
                                         const uint32_t* c2, uint32_t* c_out, size_t count, int mem) {
    if (!c || !n || !c1 || !c2 || !c_out) return tecdsa_fail(TECDSA_E_ARG, "paillier_add: null argument");
    STAGE_PROLOGUE("paillier_add", count);
    const uint32_t *d1 = S.in(c1, count * 128), *d2 = S.in(c2, count * 128);
    uint32_t* dc = S.out(c_out, count * 128);
    if (S.err) return S.err;
    Operand N, ND;
    RUN(stage_caller_key(S, n, key_idx, n_keys, count, N, ND));
    Launches L;
    add_nn(L.e128, (int)count, N, ND, 0, NONE, NONE, 0, NONE, NONE, 0, 2, arr(d1, 128), arr(d2, 128), dc, 128);
    RUN(run_nn(c, L.e128));
    return S.finish();
}

extern "C" int tecdsa_paillier_decrypt_batch(tecdsa_ctx* c, const tecdsa_keyset* ks, const uint32_t* key_row, const uint32_t* ct,
                                             uint32_t* m_out, size_t count, int mem) {
    if (!c || !ks || !key_row || !ct || !m_out) return tecdsa_fail(TECDSA_E_ARG, "paillier_decrypt: null argument");
    STAGE_PROLOGUE("paillier_decrypt", count);
    const uint32_t *dr = S.in(key_row, count), *dct = S.in(ct, count * 128);
    uint32_t* dm = S.out(m_out, count * 64);
    uint32_t *dp = S.tmp<uint32_t>(count * 64), *dq = S.tmp<uint32_t>(count * 64);
    if (S.err) return S.err;
    Launches L;
    add_decrypt(L.e128, (int)count, ks, dr, dct, dp, dq);
    RUN(run_nn(c, L.e128, 32));
    k_decrypt_finish<<<grid_for(count), 64, 0, c->stream>>>(key_arena(ks), dm, dp, dq, dr, (int)count);
    KCHECK();
    return S.finish();
}

// ------------------------------------------------------------------------------------------ L2: MtA range proof (Alice)
// AliceProof::generate on device-resident arrays (shared by the L2 entry point, tecdsa_mta_message_a_batch and the general offline stage)
int tecdsa::alice_generate_step(tecdsa_ctx* c, Stage& S, const tecdsa_keyset* ks, int n, const uint32_t* er, const uint32_t* sr, const uint32_t* da,
                              const uint32_t* dc, const uint32_t* dr, const uint32_t* dal, const uint32_t* dbe, const uint32_t* dga, const uint32_t* dro,
                              uint32_t* dz, uint32_t* de, uint32_t* ds, uint32_t* ds1, uint32_t* ds2) {
    const size_t count = (size_t)n;
    uint32_t *lin = S.tmp<uint32_t>(count * 128), *u = S.tmp<uint32_t>(count * 128), *w = S.tmp<uint32_t>(count * 64);
    if (S.err) return S.err;
    Arena A = key_arena(ks);
    k_lin<<<grid_for(count), 64, 0, c->stream>>>(lin, dal, 24, ks->tab[KT_N], er, n);
    c->count_launch();
    Launches L;
    add_nn(L.e128, n, key_n(ks, er), key_nadic(ks, er), 1, arr(dbe, 64), tab(ks->tab[KT_N], er, 64), 64, NONE, NONE, 0, 1, arr(lin, 128), NONE, u, 128);  // u (:53-55)
    add_fb(L.e64, n, ks, sr, arr(dga, 88), 88, arr(dal, 24), 24, 0, NONE, w);       // w = h1^alpha h2^gamma (:56-57)
    add_fb(L.e64, n, ks, sr, arr(dro, 72), 72, arr(da, 8), 8, 0, NONE, dz);         // z = h1^a h2^ro       (:52)
    int rc = run_nn(c, L.e128); if (rc) return rc;
    rc = run(c, L.e64, 64); if (rc) return rc;
    k_alice_mid<<<grid_for(count), 64, 0, c->stream>>>(A, er, dc, dz, u, w, da, dal, dga, dro, de, ds1, ds2, n);
    c->count_launch();
    add_exp(L.e64, 64, n, tab(ks->tab[KT_N], er, 64), 1, arr(dr, 64), arr(de, 8), 8, NONE, NONE, 0, 1, arr(dbe, 64), NONE, ds, 64);   // s = r^e beta mod N (:86)
    rc = run(c, L.e64, 64); if (rc) return rc;
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? 0 : tecdsa_fail(TECDSA_E_CUDA, "alice_generate", e);
}

extern "C" int tecdsa_alice_proof_generate_batch(tecdsa_ctx* c, const tecdsa_keyset* ks, const uint32_t* ek_row, const uint32_t* st_row,
                                                 const uint32_t* a, const uint32_t* cipher, const uint32_t* r, const uint32_t* alpha,
                                                 const uint32_t* beta, const uint32_t* gamma, const uint32_t* rho, uint32_t* z, uint32_t* e,
                                                 uint32_t* s, uint32_t* s1, uint32_t* s2, size_t count, int mem) {
    if (!c || !ks || !ek_row || !st_row || !a || !cipher || !r || !alpha || !beta || !gamma || !rho || !z || !e || !s || !s1 || !s2)
        return tecdsa_fail(TECDSA_E_ARG, "alice_proof_generate: null argument");
    STAGE_PROLOGUE("alice_proof_generate", count);
    const uint32_t *er = S.in(ek_row, count), *sr = S.in(st_row, count), *da = S.in(a, count * 8), *dc = S.in(cipher, count * 128),
                   *dr = S.in(r, count * 64), *dal = S.in(alpha, count * 24), *dbe = S.in(beta, count * 64), *dga = S.in(gamma, count * 88),
                   *dro = S.in(rho, count * 72);
    uint32_t *dz = S.out(z, count * 64), *de = S.out(e, count * 8), *ds = S.out(s, count * 64), *ds1 = S.out(s1, count * 28), *ds2 = S.out(s2, count * 92);
    if (S.err) return S.err;
    RUN(alice_generate_step(c, S, ks, (int)count, er, sr, da, dc, dr, dal, dbe, dga, dro, dz, de, ds, ds1, ds2));
    return S.finish();
}

// AliceProof::verify on device-resident arrays (shared by the L2 entry point, tecdsa_mta_message_b_batch and the general offline stage)
int tecdsa::alice_verify_step(tecdsa_ctx* c, Stage& S, const tecdsa_keyset* ks, int n, const uint32_t* er, const uint32_t* sr, const uint32_t* dc,
                            const uint32_t* dz, const uint32_t* de, const uint32_t* ds, const uint32_t* ds1, const uint32_t* ds2, uint8_t* dst) {
    const size_t count = (size_t)n;
    uint32_t *gs1 = S.tmp<uint32_t>(count * 128), *ze = S.tmp<uint32_t>(count * 64), *ce = S.tmp<uint32_t>(count * 128),
             *zei = S.tmp<uint32_t>(count * 64), *cei = S.tmp<uint32_t>(count * 128), *w = S.tmp<uint32_t>(count * 64),
             *u = S.tmp<uint32_t>(count * 128), *e2 = S.tmp<uint32_t>(count * 8);
    uint8_t *bad = S.tmp<uint8_t>(count), *okz = S.tmp<uint8_t>(count), *okc = S.tmp<uint8_t>(count);
    if (S.err) return S.err;
    Arena A = key_arena(ks);
    k_alice_vpre<<<grid_for(count), 64, 0, c->stream>>>(A, er, ds1, gs1, bad, n);
    c->count_launch();
    Launches L;
    Operand NT = tab(ks->tab[KT_NT], sr, 64), NN = tab(ks->tab[KT_NN], er, 128);
    add_exp(L.e64, 64, n, NT, 1, arr(dz, 64), arr(de, 8), 8, NONE, NONE, 0, 0, NONE, NONE, ze, 64);            // z^e (:122)
    add_nn(L.e128, n, key_n(ks, er), key_nadic(ks, er), 1, arr(dc, 128), arr(de, 8), 8, NONE, NONE, 0, 0, NONE, NONE, ce, 128);        // c^e (:135)
    int rc = run_nn(c, L.e128); if (rc) return rc;
    rc = run(c, L.e64, 64); if (rc) return rc;
    add_inv(L.i64, 64, n, NT, arr(ze, 64), zei, okz);
    add_inv(L.i128, 128, n, NN, arr(ce, 128), cei, okc);
    rc = run(c, L.i128, 128); if (rc) return rc;
    rc = run(c, L.i64, 64); if (rc) return rc;
    add_fb(L.e64, n, ks, sr, arr(ds2, 92), 92, arr(ds1, 28), 28, 1, arr(zei, 64), w);                             // w' (:129-132)
    add_nn(L.e128, n, key_n(ks, er), key_nadic(ks, er), 1, arr(ds, 64), tab(ks->tab[KT_N], er, 64), 64, NONE, NONE, 0, 2, arr(gs1, 128), arr(cei, 128), u, 128);   // u' (:141)
    rc = run_nn(c, L.e128); if (rc) return rc;
    rc = run(c, L.e64, 64); if (rc) return rc;
    k_alice_vpost<<<grid_for(count), 64, 0, c->stream>>>(A, er, dc, dz, u, w, de, bad, okz, okc, e2, dst, n);
    c->count_launch();
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? 0 : tecdsa_fail(TECDSA_E_CUDA, "alice_verify", e);
}

extern "C" int tecdsa_alice_proof_verify_batch(tecdsa_ctx* c, const tecdsa_keyset* ks, const uint32_t* ek_row, const uint32_t* st_row,
                                               const uint32_t* cipher, const uint32_t* z, const uint32_t* e, const uint32_t* s,
                                               const uint32_t* s1, const uint32_t* s2, uint8_t* status, size_t count, int mem) {
    if (!c || !ks || !ek_row || !st_row || !cipher || !z || !e || !s || !s1 || !s2 || !status)
        return tecdsa_fail(TECDSA_E_ARG, "alice_proof_verify: null argument");
    STAGE_PROLOGUE("alice_proof_verify", count);
    const uint32_t *er = S.in(ek_row, count), *sr = S.in(st_row, count), *dc = S.in(cipher, count * 128), *dz = S.in(z, count * 64),
                   *de = S.in(e, count * 8), *ds = S.in(s, count * 64), *ds1 = S.in(s1, count * 28), *ds2 = S.in(s2, count * 92);
    uint8_t* dst = S.out(status, count);
    if (S.err) return S.err;
    RUN(alice_verify_step(c, S, ks, (int)count, er, sr, dc, dz, de, ds, ds1, ds2, dst));
    return S.finish();
}

// ------------------------------------------------------------------------------------------ L2: PDL with slack
extern "C" int tecdsa_pdl_prove_batch(tecdsa_ctx* c, const tecdsa_keyset* ks, const uint32_t* ek_row, const uint32_t* st_row, const uint32_t* x,
                                      const uint32_t* r, const uint32_t* cipher, const uint32_t* Qp, const uint32_t* Gp, const uint32_t* alpha,
                                      const uint32_t* beta, const uint32_t* rho, const uint32_t* gamma, uint32_t* z, uint32_t* u1, uint32_t* u2,
                                      uint32_t* u3, uint32_t* s1, uint32_t* s2, uint32_t* s3, size_t count, int mem) {
    if (!c || !ks || !ek_row || !st_row || !x || !r || !cipher || !Qp || !Gp || !alpha || !beta || !rho || !gamma || !z || !u1 || !u2 || !u3 || !s1 || !s2 || !s3)
        return tecdsa_fail(TECDSA_E_ARG, "pdl_prove: null argument");
    STAGE_PROLOGUE("pdl_prove", count);
    const int n = (int)count;
    const uint32_t *er = S.in(ek_row, count), *sr = S.in(st_row, count), *dx = S.in(x, count * 8), *dr = S.in(r, count * 64), *dc = S.in(cipher, count * 128),
                   *dQ = S.in(Qp, count * 16), *dG = S.in(Gp, count * 16), *dal = S.in(alpha, count * 24), *dbe = S.in(beta, count * 64),
                   *dro = S.in(rho, count * 72), *dga = S.in(gamma, count * 88);
    uint32_t *dz = S.out(z, count * 64), *du1 = S.out(u1, count * 16), *du2 = S.out(u2, count * 128), *du3 = S.out(u3, count * 64),
             *ds1 = S.out(s1, count * 28), *ds2 = S.out(s2, count * 64), *ds3 = S.out(s3, count * 92);
    if (S.err) return S.err;
    RUN(pdl_prove_step(c, S, ks, n, er, sr, dx, dr, dc, dQ, dG, dal, dbe, dro, dga, dz, du1, du2, du3, ds1, ds2, ds3));
    return S.finish();
}

// PDLwSlackProof::prove on device-resident arrays
int tecdsa::pdl_prove_step(tecdsa_ctx* c, Stage& S, const tecdsa_keyset* ks, int n, const uint32_t* er, const uint32_t* sr, const uint32_t* dx, const uint32_t* dr,
                   const uint32_t* dc, const uint32_t* dQ, const uint32_t* dG, const uint32_t* dal, const uint32_t* dbe, const uint32_t* dro,
                   const uint32_t* dga, uint32_t* dz, uint32_t* du1, uint32_t* du2, uint32_t* du3, uint32_t* ds1, uint32_t* ds2, uint32_t* ds3) {
    const size_t count = (size_t)n;
    uint32_t *lin = S.tmp<uint32_t>(count * 128), *e = S.tmp<uint32_t>(count * 8);
    if (S.err) return S.err;
    Arena A = key_arena(ks);
    k_pdl_pre<<<grid_for(count), 64, 0, c->stream>>>(A, er, dG, dal, du1, lin, n);
    KCHECK();
    Launches L;
    add_fb(L.e64, n, ks, sr, arr(dro, 72), 72, arr(dx, 8), 8, 0, NONE, dz);                 // z  = h1^x h2^rho       (:78-84)
    add_fb(L.e64, n, ks, sr, arr(dga, 88), 88, arr(dal, 24), 24, 0, NONE, du3);             // u3 = h1^alpha h2^gamma (:93-99)
    add_nn(L.e128, n, key_n(ks, er), key_nadic(ks, er), 1, arr(dbe, 64), tab(ks->tab[KT_N], er, 64), 64, NONE, NONE, 0, 1, arr(lin, 128), NONE, du2, 128);   // u2 (:86-92)
    RUN(run_nn(c, L.e128)); RUN(run(c, L.e64, 64));
    k_pdl_mid<<<grid_for(count), 64, 0, c->stream>>>(dG, dQ, dc, dz, du1, du2, du3, dx, dal, dro, dga, e, ds1, ds3, n);
    KCHECK();
    add_exp(L.e64, 64, n, tab(ks->tab[KT_N], er, 64), 1, arr(dr, 64), arr(e, 8), 8, NONE, NONE, 0, 1, arr(dbe, 64), NONE, ds2, 64);   // s2 = r^e beta mod N (:113)
    RUN(run(c, L.e64, 64));
    return 0;
}

extern "C" int tecdsa_pdl_verify_batch(tecdsa_ctx* c, const tecdsa_keyset* ks, const uint32_t* ek_row, const uint32_t* st_row, const uint32_t* cipher,
                                       const uint32_t* Qp, const uint32_t* Gp, const uint32_t* z, const uint32_t* u1, const uint32_t* u2,
                                       const uint32_t* u3, const uint32_t* s1, const uint32_t* s2, const uint32_t* s3, uint8_t* status, size_t count, int mem) {
    if (!c || !ks || !ek_row || !st_row || !cipher || !Qp || !Gp || !z || !u1 || !u2 || !u3 || !s1 || !s2 || !s3 || !status)
        return tecdsa_fail(TECDSA_E_ARG, "pdl_verify: null argument");
    STAGE_PROLOGUE("pdl_verify", count);
    const int n = (int)count;
    const uint32_t *er = S.in(ek_row, count), *sr = S.in(st_row, count), *dc = S.in(cipher, count * 128), *dQ = S.in(Qp, count * 16), *dG = S.in(Gp, count * 16),
                   *dz = S.in(z, count * 64), *du1 = S.in(u1, count * 16), *du2 = S.in(u2, count * 128), *du3 = S.in(u3, count * 64),
                   *ds1 = S.in(s1, count * 28), *ds2 = S.in(s2, count * 64), *ds3 = S.in(s3, count * 92);
    uint8_t* dst = S.out(status, count);
    if (S.err) return S.err;
    RUN(pdl_verify_step(c, S, ks, n, er, sr, dc, dQ, dG, dz, du1, du2, du3, ds1, ds2, ds3, dst));
    return S.finish();
}

// PDLwSlackProof::verify on device-resident arrays
int tecdsa::pdl_verify_step(tecdsa_ctx* c, Stage& S, const tecdsa_keyset* ks, int n, const uint32_t* er, const uint32_t* sr, const uint32_t* dc, const uint32_t* dQ,
                    const uint32_t* dG, const uint32_t* dz, const uint32_t* du1, const uint32_t* du2, const uint32_t* du3, const uint32_t* ds1,
                    const uint32_t* ds2, const uint32_t* ds3, uint8_t* dst) {
    const size_t count = (size_t)n;
    uint32_t *e = S.tmp<uint32_t>(count * 8), *lin = S.tmp<uint32_t>(count * 128), *ze = S.tmp<uint32_t>(count * 64), *ce = S.tmp<uint32_t>(count * 128),
             *zei = S.tmp<uint32_t>(count * 64), *cei = S.tmp<uint32_t>(count * 128), *u2t = S.tmp<uint32_t>(count * 128), *u3t = S.tmp<uint32_t>(count * 64);
    uint8_t *okz = S.tmp<uint8_t>(count), *okc = S.tmp<uint8_t>(count);
    if (S.err) return S.err;
    Arena A = key_arena(ks);
    k_pdl_vpre<<<grid_for(count), 64, 0, c->stream>>>(A, er, dG, dQ, dc, dz, du1, du2, du3, ds1, e, lin, n);
    KCHECK();
    Launches L;
    Operand NT = tab(ks->tab[KT_NT], sr, 64), NN = tab(ks->tab[KT_NN], er, 128);
    add_exp(L.e64, 64, n, NT, 1, arr(dz, 64), arr(e, 8), 8, NONE, NONE, 0, 0, NONE, NONE, ze, 64);          // z^e; (z^-1)^e == (z^e)^-1
    add_nn(L.e128, n, key_n(ks, er), key_nadic(ks, er), 1, arr(dc, 128), arr(e, 8), 8, NONE, NONE, 0, 0, NONE, NONE, ce, 128);      // c^e
    RUN(run_nn(c, L.e128)); RUN(run(c, L.e64, 64));
    add_inv(L.i64, 64, n, NT, arr(ze, 64), zei, okz);
    add_inv(L.i128, 128, n, NN, arr(ce, 128), cei, okc);
    RUN(run(c, L.i128, 128)); RUN(run(c, L.i64, 64));
    add_fb(L.e64, n, ks, sr, arr(ds3, 92), 92, arr(ds1, 28), 28, 1, arr(zei, 64), u3t);                        // u3' (:158-172)
    add_nn(L.e128, n, key_n(ks, er), key_nadic(ks, er), 1, arr(ds2, 64), tab(ks->tab[KT_N], er, 64), 64, NONE, NONE, 0, 2, arr(lin, 128), arr(cei, 128), u2t, 128);   // u2' (:144-157)
    RUN(run_nn(c, L.e128)); RUN(run(c, L.e64, 64));
    k_pdl_vpost<<<grid_for(count), 64, 0, c->stream>>>(dG, dQ, du1, du2, du3, ds1, e, u2t, u3t, okz, okc, dst, n);
    KCHECK();
    return 0;
}

// ------------------------------------------------------------------------------------------ L2: Bob's range proof (MtA / MtAwc)
extern "C" int tecdsa_bob_proof_generate_batch(tecdsa_ctx* c, const tecdsa_keyset* ks, const uint32_t* ek_row, const uint32_t* st_row, int check,
                                               const uint32_t* a_enc, const uint32_t* mta_enc, const uint32_t* b, const uint32_t* beta_prim,
                                               const uint32_t* r, const uint32_t* alpha, const uint32_t* beta, const uint32_t* gamma,
                                               const uint32_t* ro, const uint32_t* ro_prim, const uint32_t* sigma, const uint32_t* tau,
                                               uint32_t* t, uint32_t* z, uint32_t* e, uint32_t* s, uint32_t* s1, uint32_t* s2, uint32_t* t1,
                                               uint32_t* t2, uint32_t* u, size_t count, int mem) {
    if (!c || !ks || !ek_row || !st_row || !a_enc || !mta_enc || !b || !beta_prim || !r || !alpha || !beta || !gamma || !ro || !ro_prim || !sigma ||
        !tau || !t || !z || !e || !s || !s1 || !s2 || !t1 || !t2 || (check && !u))
        return tecdsa_fail(TECDSA_E_ARG, "bob_proof_generate: null argument");
    STAGE_PROLOGUE("bob_proof_generate", count);
    const int n = (int)count;
    const uint32_t *er = S.in(ek_row, count), *sr = S.in(st_row, count), *da = S.in(a_enc, count * 128), *dm = S.in(mta_enc, count * 128),
                   *db = S.in(b, count * 8), *dbp = S.in(beta_prim, count * 64), *dr = S.in(r, count * 64), *dal = S.in(alpha, count * 24),
                   *dbe = S.in(beta, count * 64), *dga = S.in(gamma, count * 80), *dro = S.in(ro, count * 72), *drp = S.in(ro_prim, count * 88),
                   *dsi = S.in(sigma, count * 72), *dta = S.in(tau, count * 88);
    uint32_t *dt = S.out(t, count * 64), *dz = S.out(z, count * 64), *de = S.out(e, count * 8), *ds = S.out(s, count * 64), *ds1 = S.out(s1, count * 28),
             *ds2 = S.out(s2, count * 92), *dt1 = S.out(t1, count * 84), *dt2 = S.out(t2, count * 92), *du = check ? S.out(u, count * 16) : nullptr;
    uint32_t *zp = S.tmp<uint32_t>(count * 64), *w = S.tmp<uint32_t>(count * 64), *v = S.tmp<uint32_t>(count * 128), *lin = S.tmp<uint32_t>(count * 128);
    if (S.err) return S.err;
    Arena A = key_arena(ks);
    k_lin_wide<<<grid_for(count), 64, 0, c->stream>>>(A, er, dga, 80, lin, n);
    KCHECK();
    Launches L;
    add_fb(L.e64, n, ks, sr, arr(dro, 72), 72, arr(db, 8), 8, 0, NONE, dz);                 // z  = h1^b h2^ro             (:238)
    add_fb(L.e64, n, ks, sr, arr(drp, 88), 88, arr(dal, 24), 24, 0, NONE, zp);              // z' = h1^alpha h2^ro'        (:239-241)
    add_fb(L.e64, n, ks, sr, arr(dsi, 72), 72, arr(dbp, 64), 64, 0, NONE, dt);              // t  = h1^beta' h2^sigma      (:242-243)
    add_fb(L.e64, n, ks, sr, arr(dta, 88), 88, arr(dga, 80), 80, 0, NONE, w);               // w  = h1^gamma h2^tau        (:244-245)
    // v = a_enc^alpha * (gamma N + 1) * beta^N mod N^2                                      (:246-249)
    add_nn(L.e128, n, key_n(ks, er), key_nadic(ks, er), 2, arr(dbe, 64), tab(ks->tab[KT_N], er, 64), 64, arr(da, 128), arr(dal, 24), 24, 1, arr(lin, 128), NONE, v, 128);
    RUN(run_nn(c, L.e128)); RUN(run(c, L.e64, 64));
    k_bob_mid<<<grid_for(count), 64, 0, c->stream>>>(A, er, check, da, dm, dz, zp, dt, v, w, db, dbp, dal, dga, dro, drp, dsi, dta, de, ds1, ds2, dt1, dt2, du, n);
    KCHECK();
    add_exp(L.e64, 64, n, tab(ks->tab[KT_N], er, 64), 1, arr(dr, 64), arr(de, 8), 8, NONE, NONE, 0, 1, arr(dbe, 64), NONE, ds, 64);   // s = r^e beta mod N (:291)
    RUN(run(c, L.e64, 64));
    return S.finish();
}

extern "C" int tecdsa_bob_proof_verify_batch(tecdsa_ctx* c, const tecdsa_keyset* ks, const uint32_t* ek_row, const uint32_t* st_row, const uint32_t* a_enc,
                                             const uint32_t* mta_out, const uint32_t* t, const uint32_t* z, const uint32_t* e, const uint32_t* s,
                                             const uint32_t* s1, const uint32_t* s2, const uint32_t* t1, const uint32_t* t2, const uint32_t* X,
                                             const uint32_t* u, uint8_t* status, size_t count, int mem) {
    if (!c || !ks || !ek_row || !st_row || !a_enc || !mta_out || !t || !z || !e || !s || !s1 || !s2 || !t1 || !t2 || !status || ((X == nullptr) != (u == nullptr)))
        return tecdsa_fail(TECDSA_E_ARG, "bob_proof_verify: bad argument");
    STAGE_PROLOGUE("bob_proof_verify", count);
    const int n = (int)count;
    const uint32_t *er = S.in(ek_row, count), *sr = S.in(st_row, count), *da = S.in(a_enc, count * 128), *dm = S.in(mta_out, count * 128), *dt = S.in(t, count * 64),
                   *dz = S.in(z, count * 64), *de = S.in(e, count * 8), *ds = S.in(s, count * 64), *ds1 = S.in(s1, count * 28), *ds2 = S.in(s2, count * 92),
                   *dt1 = S.in(t1, count * 84), *dt2 = S.in(t2, count * 92), *dX = S.in(X, count * 16), *dU = S.in(u, count * 16);
    uint8_t* dst = S.out(status, count);
    uint32_t *ze = S.tmp<uint32_t>(count * 64), *te = S.tmp<uint32_t>(count * 64), *me = S.tmp<uint32_t>(count * 128), *zei = S.tmp<uint32_t>(count * 64),
             *tei = S.tmp<uint32_t>(count * 64), *mei = S.tmp<uint32_t>(count * 128), *lin = S.tmp<uint32_t>(count * 128), *zp = S.tmp<uint32_t>(count * 64),
             *w = S.tmp<uint32_t>(count * 64), *v = S.tmp<uint32_t>(count * 128), *e2 = S.tmp<uint32_t>(count * 8);
    uint8_t *bad = S.tmp<uint8_t>(count), *ok1 = S.tmp<uint8_t>(count), *ok2 = S.tmp<uint8_t>(count), *ok3 = S.tmp<uint8_t>(count);
    if (S.err) return S.err;
    Arena A = key_arena(ks);
    k_bob_vpre<<<grid_for(count), 64, 0, c->stream>>>(ds1, bad, n);
    KCHECK();
    k_lin_wide<<<grid_for(count), 64, 0, c->stream>>>(A, er, dt1, 84, lin, n);
    KCHECK();
    Launches L;
    Operand NT = tab(ks->tab[KT_NT], sr, 64), NN = tab(ks->tab[KT_NN], er, 128);
    add_exp(L.e64, 64, n, NT, 1, arr(dz, 64), arr(de, 8), 8, NONE, NONE, 0, 0, NONE, NONE, ze, 64);           // z^e   (:339)
    add_exp(L.e64, 64, n, NT, 1, arr(dt, 64), arr(de, 8), 8, NONE, NONE, 0, 0, NONE, NONE, te, 64);           // t^e   (:363)
    add_nn(L.e128, n, key_n(ks, er), key_nadic(ks, er), 1, arr(dm, 128), arr(de, 8), 8, NONE, NONE, 0, 0, NONE, NONE, me, 128);       // mta^e (:351)
    RUN(run_nn(c, L.e128)); RUN(run(c, L.e64, 64));
    add_inv(L.i64, 64, n, NT, arr(ze, 64), zei, ok1);
    add_inv(L.i64, 64, n, NT, arr(te, 64), tei, ok3);
    add_inv(L.i128, 128, n, NN, arr(me, 128), mei, ok2);
    RUN(run(c, L.i128, 128)); RUN(run(c, L.i64, 64));
    add_fb(L.e64, n, ks, sr, arr(ds2, 92), 92, arr(ds1, 28), 28, 1, arr(zei, 64), zp);                          // z' (:346-349)
    add_fb(L.e64, n, ks, sr, arr(dt2, 92), 92, arr(dt1, 84), 84, 1, arr(tei, 64), w);                           // w  (:369-372)
    // v = a_enc^s1 * s^N * (t1 N + 1) * (mta^e)^-1 mod N^2                                                      (:357-361)
    add_nn(L.e128, n, key_n(ks, er), key_nadic(ks, er), 2, arr(ds, 64), tab(ks->tab[KT_N], er, 64), 64, arr(da, 128), arr(ds1, 28), 28, 2, arr(lin, 128), arr(mei, 128), v, 128);
    RUN(run_nn(c, L.e128)); RUN(run(c, L.e64, 64));
    k_bob_vpost<<<grid_for(count), 64, 0, c->stream>>>(A, er, da, dm, dz, zp, dt, v, w, de, ds1, dX, dU, bad, ok1, ok2, ok3, e2, dst, n);
    KCHECK();
    return S.finish();
}


// ------------------------------------------------------------------------------------------ curv sigma proofs / hashes
extern "C" int tecdsa_dlog_prove_batch(tecdsa_ctx* c, const uint32_t* sk, const uint32_t* nonce, uint32_t* proof, size_t count, int mem) {
    if (!sk || !nonce || !proof) return tecdsa_fail(TECDSA_E_ARG, "dlog_prove: null argument");
    STAGE_PROLOGUE("dlog_prove", count);
    const uint32_t *a = S.in(sk, count * 8), *b = S.in(nonce, count * 8);
    uint32_t* o = S.out(proof, count * 40);
    if (S.err) return S.err;
    k_dlog_prove<<<grid_for(count), 64, 0, c->stream>>>(o, a, b, (int)count);
    KCHECK();
    return S.finish();
}
extern "C" int tecdsa_dlog_verify_batch(tecdsa_ctx* c, const uint32_t* proof, uint8_t* status, size_t count, int mem) {
    if (!proof || !status) return tecdsa_fail(TECDSA_E_ARG, "dlog_verify: null argument");
    STAGE_PROLOGUE("dlog_verify", count);
    const uint32_t* a = S.in(proof, count * 40);
    uint8_t* o = S.out(status, count);
    if (S.err) return S.err;
    k_dlog_verify<<<grid_for(count), 64, 0, c->stream>>>(a, o, (int)count);
    KCHECK();
    return S.finish();
}
extern "C" int tecdsa_pedersen_prove_batch(tecdsa_ctx* c, const uint32_t* m, const uint32_t* r, const uint32_t* s1, const uint32_t* s2,
                                           uint32_t* com, uint32_t* proof, size_t count, int mem) {
    if (!m || !r || !s1 || !s2 || !com || !proof) return tecdsa_fail(TECDSA_E_ARG, "pedersen_prove: null argument");
    STAGE_PROLOGUE("pedersen_prove", count);
    const uint32_t *dm = S.in(m, count * 8), *dr = S.in(r, count * 8), *d1 = S.in(s1, count * 8), *d2 = S.in(s2, count * 8);
    uint32_t *dc = S.out(com, count * 16), *dp = S.out(proof, count * 64);
    if (S.err) return S.err;
    RUN(pedersen_prove_step(c, (int)count, dm, dr, d1, d2, dc, dp));
    return S.finish();
}
int tecdsa::pedersen_prove_step(tecdsa_ctx* c, int n, const uint32_t* m, const uint32_t* r, const uint32_t* s1, const uint32_t* s2, uint32_t* com, uint32_t* proof) {
    k_pedersen_prove<<<grid_for((size_t)n), 64, 0, c->stream>>>(com, proof, m, r, s1, s2, n);
    KCHECK();
    return 0;
}
extern "C" int tecdsa_pedersen_verify_batch(tecdsa_ctx* c, const uint32_t* com, const uint32_t* proof, uint8_t* status, size_t count, int mem) {
    if (!com || !proof || !status) return tecdsa_fail(TECDSA_E_ARG, "pedersen_verify: null argument");
    STAGE_PROLOGUE("pedersen_verify", count);
    const uint32_t *dc = S.in(com, count * 16), *dp = S.in(proof, count * 64);
    uint8_t* o = S.out(status, count);
    if (S.err) return S.err;
    RUN(pedersen_verify_step(c, (int)count, dc, dp, o));
    return S.finish();
}
int tecdsa::pedersen_verify_step(tecdsa_ctx* c, int n, const uint32_t* com, const uint32_t* proof, uint8_t* status) {
    k_pedersen_verify<<<grid_for((size_t)n), 64, 0, c->stream>>>(com, proof, status, n);
    KCHECK();
    return 0;
}
extern "C" int tecdsa_heg_prove_batch(tecdsa_ctx* c, const uint32_t* G, const uint32_t* D, const uint32_t* E, const uint32_t* x, const uint32_t* r,
                                      const uint32_t* s1, const uint32_t* s2, uint32_t* proof, size_t count, int mem) {
    if (!G || !D || !E || !x || !r || !s1 || !s2 || !proof) return tecdsa_fail(TECDSA_E_ARG, "heg_prove: null argument");
    STAGE_PROLOGUE("heg_prove", count);
    const uint32_t *dG = S.in(G, count * 16), *dD = S.in(D, count * 16), *dE = S.in(E, count * 16), *dx = S.in(x, count * 8), *dr = S.in(r, count * 8),
                   *d1 = S.in(s1, count * 8), *d2 = S.in(s2, count * 8);
    uint32_t* o = S.out(proof, count * 48);
    if (S.err) return S.err;
    RUN(heg_prove_step(c, (int)count, dG, dD, dE, dx, dr, d1, d2, o));
    return S.finish();
}
int tecdsa::heg_prove_step(tecdsa_ctx* c, int n, const uint32_t* G, const uint32_t* D, const uint32_t* E, const uint32_t* x, const uint32_t* r, const uint32_t* s1,
                   const uint32_t* s2, uint32_t* proof) {
    k_heg_prove<<<grid_for((size_t)n), 64, 0, c->stream>>>(proof, G, D, E, x, r, s1, s2, n);
    KCHECK();
    return 0;
}
extern "C" int tecdsa_heg_verify_batch(tecdsa_ctx* c, const uint32_t* G, const uint32_t* D, const uint32_t* E, const uint32_t* proof, uint8_t* status,
                                       size_t count, int mem) {
    if (!G || !D || !E || !proof || !status) return tecdsa_fail(TECDSA_E_ARG, "heg_verify: null argument");
    STAGE_PROLOGUE("heg_verify", count);
    const uint32_t *dG = S.in(G, count * 16), *dD = S.in(D, count * 16), *dE = S.in(E, count * 16), *dp = S.in(proof, count * 48);
    uint8_t* o = S.out(status, count);
    if (S.err) return S.err;
    RUN(heg_verify_step(c, (int)count, dG, dD, dE, dp, o));
    return S.finish();
}
int tecdsa::heg_verify_step(tecdsa_ctx* c, int n, const uint32_t* G, const uint32_t* D, const uint32_t* E, const uint32_t* proof, uint8_t* status) {
    k_heg_verify<<<grid_for((size_t)n), 64, 0, c->stream>>>(proof, G, D, E, status, n);
    KCHECK();
    return 0;
}
extern "C" int tecdsa_sha256_bigints_batch(tecdsa_ctx* c, const uint32_t* data, const int* item_limbs, int n_items, uint32_t* digest, size_t count, int mem) {
    if (!data || !item_limbs || !digest || n_items <= 0 || n_items > 64) return tecdsa_fail(TECDSA_E_ARG, "sha256_bigints: bad argument");
    STAGE_PROLOGUE("sha256_bigints", count);
    int stride = 0;
    for (int j = 0; j < n_items; j++) { if (item_limbs[j] <= 0) { return tecdsa_fail(TECDSA_E_ARG, "sha256_bigints: bad item size"); } stride += item_limbs[j]; }
    const uint32_t* dd = S.in(data, count * (size_t)stride);
    int* dl = S.tmp<int>(n_items);
    uint32_t* o = S.out(digest, count * 8);
    if (S.err) return S.err;
    if (cudaMemcpyAsync(dl, item_limbs, n_items * sizeof(int), cudaMemcpyHostToDevice, c->stream) != cudaSuccess) return tecdsa_fail(TECDSA_E_CUDA, "copy");
    k_sha256_bigints<<<grid_for(count), 64, 0, c->stream>>>(dd, stride, dl, n_items, o, (int)count);
    KCHECK();
    return S.finish();
}
extern "C" int tecdsa_hash_commitment_batch(tecdsa_ctx* c, const uint32_t* points, const uint32_t* blind, uint32_t* com, size_t count, int mem) {
    if (!points || !blind || !com) return tecdsa_fail(TECDSA_E_ARG, "hash_commitment: null argument");
    STAGE_PROLOGUE("hash_commitment", count);
    const uint32_t *dp = S.in(points, count * 16), *db = S.in(blind, count * 8);
    uint32_t* o = S.out(com, count * 8);
    if (S.err) return S.err;
    RUN(hash_commitment_step(c, (int)count, dp, db, o));
    return S.finish();
}
int tecdsa::hash_commitment_step(tecdsa_ctx* c, int n, const uint32_t* points, const uint32_t* blind, uint32_t* com) {
    k_hash_commit<<<grid_for((size_t)n), 64, 0, c->stream>>>(points, blind, com, n);
    KCHECK();
    return 0;
}


// ------------------------------------------------------------------------------------------ L2: MtA messages
extern "C" int tecdsa_mta_message_a_batch(tecdsa_ctx* c, const tecdsa_keyset* ks, const uint32_t* ek_row, const uint32_t* st_rows, int n_st,
                                          const uint32_t* a, const uint32_t* r, const uint32_t* alpha, const uint32_t* beta, const uint32_t* gamma,
                                          const uint32_t* rho, uint32_t* c_out, uint32_t* z, uint32_t* e, uint32_t* s, uint32_t* s1, uint32_t* s2,
                                          size_t count, int mem) {
    if (!c || !ks || !ek_row || !a || !r || !c_out || n_st < 0 || n_st > 16) return tecdsa_fail(TECDSA_E_ARG, "mta_message_a: bad argument");
    if (n_st > 0 && (!st_rows || !alpha || !beta || !gamma || !rho || !z || !e || !s || !s1 || !s2)) return tecdsa_fail(TECDSA_E_ARG, "mta_message_a: null proof buffer");
    STAGE_PROLOGUE("mta_message_a", count);
    const size_t np = count * (size_t)n_st;
    const uint32_t *er = S.in(ek_row, count), *da = S.in(a, count * 8), *dr = S.in(r, count * 64);
    uint32_t* dc = S.out(c_out, count * 128);
    const uint32_t *sr = S.in(st_rows, np), *dal = S.in(alpha, np * 24), *dbe = S.in(beta, np * 64), *dga = S.in(gamma, np * 88), *dro = S.in(rho, np * 72);
    uint32_t *dz = S.out(z, np * 64), *de = S.out(e, np * 8), *ds = S.out(s, np * 64), *ds1 = S.out(s1, np * 28), *ds2 = S.out(s2, np * 92);
    if (S.err) return S.err;
    RUN(mta_message_a_step(c, S, ks, (int)count, n_st, er, da, dr, sr, dal, dbe, dga, dro, dc, dz, de, ds, ds1, ds2));
    return S.finish();
}

// c = Enc(a; r) = (1 + a N) r^N mod N^2 under key rows er (mod.rs:68-75), on device-resident arrays
int tecdsa::mta_encrypt_step(tecdsa_ctx* c, Stage& S, const tecdsa_keyset* ks, int n, const uint32_t* er, const uint32_t* da, const uint32_t* dr, uint32_t* dc) {
    const size_t count = (size_t)n;
    uint32_t *a64 = S.tmp<uint32_t>(count * 64), *lin = S.tmp<uint32_t>(count * 128);
    if (S.err) return S.err;
    CK(cudaMemsetAsync(a64, 0, count * 64 * 4, c->stream));
    CK(cudaMemcpy2DAsync(a64, 64 * 4, da, 8 * 4, 8 * 4, count, cudaMemcpyDeviceToDevice, c->stream));
    k_lin<<<grid_for(count), 64, 0, c->stream>>>(lin, a64, 64, ks->tab[KT_N], er, n);
    KCHECK();
    Launches L;
    add_nn(L.e128, n, key_n(ks, er), key_nadic(ks, er), 1, arr(dr, 64), tab(ks->tab[KT_N], er, 64), 64, NONE, NONE, 0, 1, arr(lin, 128), NONE, dc, 128);
    RUN(run_nn(c, L.e128));
    return 0;
}

// MessageA::a (mod.rs:52-80) on device-resident arrays: c, and one AliceProof per (instance, statement), instance-major
int tecdsa::mta_message_a_step(tecdsa_ctx* c, Stage& S, const tecdsa_keyset* ks, int n, int n_st, const uint32_t* er, const uint32_t* da, const uint32_t* dr,
                       const uint32_t* sr, const uint32_t* dal, const uint32_t* dbe, const uint32_t* dga, const uint32_t* dro, uint32_t* dc, uint32_t* dz,
                       uint32_t* de, uint32_t* ds, uint32_t* ds1, uint32_t* ds2) {
    const size_t count = (size_t)n, np = count * (size_t)n_st;
    RUN(mta_encrypt_step(c, S, ks, n, er, da, dr, dc));
    if (n_st > 0) {
        uint32_t *er_f = S.tmp<uint32_t>(np), *a_f = S.tmp<uint32_t>(np * 8), *r_f = S.tmp<uint32_t>(np * 64), *c_f = S.tmp<uint32_t>(np * 128);
        if (S.err) return S.err;
        const int g = grid_for(np);
        k_expand<<<g, 64, 0, c->stream>>>(er_f, er, 1, n_st, n);
        k_expand<<<g, 64, 0, c->stream>>>(a_f, da, 8, n_st, n);
        k_expand<<<g, 64, 0, c->stream>>>(r_f, dr, 64, n_st, n);
        k_expand<<<g, 64, 0, c->stream>>>(c_f, dc, 128, n_st, n);
        KCHECK();
        RUN(alice_generate_step(c, S, ks, (int)np, er_f, sr, a_f, c_f, r_f, dal, dbe, dga, dro, dz, de, ds, ds1, ds2));
    }
    return 0;
}

extern "C" int tecdsa_mta_message_b_batch(tecdsa_ctx* c, const tecdsa_keyset* ks, const uint32_t* ek_row, const uint32_t* st_rows, int n_st,
                                          const uint32_t* b, const uint32_t* c_a, const uint32_t* z, const uint32_t* e, const uint32_t* s,
                                          const uint32_t* s1, const uint32_t* s2, const uint32_t* randomness, const uint32_t* beta_tag,
                                          const uint32_t* nonce_b, const uint32_t* nonce_beta, uint32_t* c_b, uint32_t* b_proof,
                                          uint32_t* beta_tag_proof, uint32_t* beta, uint8_t* status, size_t count, int mem) {
    if (!c || !ks || !ek_row || !b || !c_a || !randomness || !beta_tag || !nonce_b || !nonce_beta || !c_b || !b_proof || !beta_tag_proof || !beta || !status ||
        n_st < 0 || n_st > 16)
        return tecdsa_fail(TECDSA_E_ARG, "mta_message_b: bad argument");
    if (n_st > 0 && (!st_rows || !z || !e || !s || !s1 || !s2)) return tecdsa_fail(TECDSA_E_ARG, "mta_message_b: null proof buffer");
    STAGE_PROLOGUE("mta_message_b", count);
    const size_t np = count * (size_t)n_st;
    const uint32_t *er = S.in(ek_row, count), *db = S.in(b, count * 8), *dca = S.in(c_a, count * 128), *dr = S.in(randomness, count * 64),
                   *dbt = S.in(beta_tag, count * 64), *dnb = S.in(nonce_b, count * 8), *dnt = S.in(nonce_beta, count * 8);
    const uint32_t *sr = S.in(st_rows, np), *dz = S.in(z, np * 64), *de = S.in(e, np * 8), *ds = S.in(s, np * 64), *ds1 = S.in(s1, np * 28), *ds2 = S.in(s2, np * 92);
    uint32_t *dcb = S.out(c_b, count * 128), *dbp = S.out(b_proof, count * 40), *dtp = S.out(beta_tag_proof, count * 40), *dbeta = S.out(beta, count * 8);
    uint8_t* dst = S.out(status, count);
    if (S.err) return S.err;
    RUN(mta_message_b_step(c, S, ks, (int)count, er, db, dca, dr, dbt, dnb, dnt, n_st, sr, dz, de, ds, ds1, ds2, nullptr, dcb, dbp, dtp, dbeta, dst));
    return S.finish();
}

// MessageB::b (mod.rs:84-148) on device-resident arrays.  The n_st range proofs of instance i's MessageA are verified here
// (instance-major, as tecdsa_mta_message_b_batch takes them), unless `checked` already holds their statuses ([n][n_st]): a caller
// that answers one MessageA several times verifies its proofs once.
int tecdsa::mta_message_b_step(tecdsa_ctx* c, Stage& S, const tecdsa_keyset* ks, int n, const uint32_t* er, const uint32_t* db, const uint32_t* dca, const uint32_t* dr,
                       const uint32_t* dbt, const uint32_t* dnb, const uint32_t* dnt, int n_st, const uint32_t* sr, const uint32_t* dz, const uint32_t* de,
                       const uint32_t* ds, const uint32_t* ds1, const uint32_t* ds2, const uint8_t* checked, uint32_t* dcb, uint32_t* dbp, uint32_t* dtp,
                       uint32_t* dbeta, uint8_t* dst) {
    const size_t count = (size_t)n, np = count * (size_t)n_st;
    uint8_t* pst = checked ? nullptr : S.tmp<uint8_t>(np ? np : 1);
    uint32_t* lin = S.tmp<uint32_t>(count * 128);
    if (S.err) return S.err;
    if (n_st > 0 && !checked) {     // verify every range proof of MessageA (mod.rs:123-131)
        uint32_t *er_f = S.tmp<uint32_t>(np), *c_f = S.tmp<uint32_t>(np * 128);
        if (S.err) return S.err;
        k_expand<<<grid_for(np), 64, 0, c->stream>>>(er_f, er, 1, n_st, n);
        k_expand<<<grid_for(np), 64, 0, c->stream>>>(c_f, dca, 128, n_st, n);
        KCHECK();
        RUN(alice_verify_step(c, S, ks, (int)np, er_f, sr, c_f, dz, de, ds, ds1, ds2, pst));
    }
    // c_b = c_a^b * Enc(beta'; r') mod N^2   (mod.rs:133-145)
    k_lin<<<grid_for(count), 64, 0, c->stream>>>(lin, dbt, 64, ks->tab[KT_N], er, n);
    KCHECK();
    Launches L;
    add_nn(L.e128, n, key_n(ks, er), key_nadic(ks, er), 2, arr(dr, 64), tab(ks->tab[KT_N], er, 64), 64, arr(dca, 128), arr(db, 8), 8, 1, arr(lin, 128), NONE, dcb, 128);
    RUN(run_nn(c, L.e128));
    k_mta_b_post<<<grid_for(count), 64, 0, c->stream>>>(checked ? checked : pst, n_st, db, dbt, dnb, dnt, dbeta, dbp, dtp, dst, n);
    KCHECK();
    return 0;
}

extern "C" int tecdsa_mta_get_alpha_batch(tecdsa_ctx* c, const tecdsa_keyset* ks, const uint32_t* dk_row, const uint32_t* a, const uint32_t* c_b,
                                          const uint32_t* b_proof, const uint32_t* beta_tag_proof, uint32_t* alpha, uint32_t* alpha_plain,
                                          uint8_t* status, size_t count, int mem) {
    if (!c || !ks || !dk_row || !a || !c_b || !b_proof || !beta_tag_proof || !alpha || !status) return tecdsa_fail(TECDSA_E_ARG, "mta_get_alpha: null argument");
    STAGE_PROLOGUE("mta_get_alpha", count);
    const uint32_t *dr = S.in(dk_row, count), *da = S.in(a, count * 8), *dcb = S.in(c_b, count * 128), *dbp = S.in(b_proof, count * 40), *dtp = S.in(beta_tag_proof, count * 40);
    uint32_t* dal = S.out(alpha, count * 8);
    uint32_t* dpl = alpha_plain ? S.out(alpha_plain, count * 64) : S.tmp<uint32_t>(count * 64);
    uint8_t* dst = S.out(status, count);
    if (S.err) return S.err;
    RUN(mta_get_alpha_step(c, S, ks, (int)count, dr, da, dcb, dbp, dtp, dal, dpl, dst));
    return S.finish();
}

// MessageB::verify_proofs_get_alpha (mod.rs:150-179) on device-resident arrays
int tecdsa::mta_get_alpha_step(tecdsa_ctx* c, Stage& S, const tecdsa_keyset* ks, int n, const uint32_t* dr, const uint32_t* da, const uint32_t* dcb, const uint32_t* dbp,
                       const uint32_t* dtp, uint32_t* dal, uint32_t* dpl, uint8_t* dst) {
    const size_t count = (size_t)n;
    uint32_t *dp = S.tmp<uint32_t>(count * 64), *dq = S.tmp<uint32_t>(count * 64);
    if (S.err) return S.err;
    Launches L;
    add_decrypt(L.e128, n, ks, dr, dcb, dp, dq);
    RUN(run_nn(c, L.e128, 32));
    k_mta_alpha<<<grid_for(count), 64, 0, c->stream>>>(key_arena(ks), dr, dp, dq, da, dbp, dtp, dpl, dal, dst, n);
    KCHECK();
    return 0;
}
