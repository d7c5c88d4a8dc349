// "Glue" kernels of the batched GG20 offline stage: everything between the big-integer job
// launches — EC arithmetic, Fiat-Shamir hashing, plain-integer responses, Paillier CRT
// recombination, the sigma proofs of curv, and the per-round checks.  One thread per unit.
// Each kernel names the reference lines it follows; paths are relative to
// /root/reference/src.
#pragma once
#include "gg20_fields.h"
#include "secp256k1.cuh"
#include "sha256.cuh"
#include "st_bigint.cuh"
#include "../../include/tecdsa_b200.h"

namespace tecdsa {

using namespace secp;

__device__ __constant__ const int KEY_SIZE_D[KT_COUNT] = {64, 128, 64, 64, 64, 64, 64, 32, 32, 32, 32, 32, 32, 32, 32, 32, 64, 32, 32, 8, 16};
// q^3 (24 limbs): the verifier's range bound `s1 > q^3 => reject` (utilities/mta/range_proofs.rs:118)
__device__ __constant__ const uint32_t Q3_LIMBS[24] = {
    0x857B73C1u, 0xEB6926B7u, 0xE1E11B11u, 0x3552090Fu, 0x7A1CF066u, 0xD9EF0F38u, 0x02D99574u, 0x46385C85u,
    0x16EA33B3u, 0xFD393075u, 0x11A63C8Cu, 0x7EF36D11u, 0x1367174Du, 0xB3C7E1ADu, 0x8553D351u, 0xD8355680u,
    0x70A2C3C7u, 0x3F771BA6u, 0x0DD9E0B3u, 0x300C96B4u, 0xFFFFFFFCu, 0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu};

struct Arena {
    uint32_t* base;
    int U;
    uint32_t off[F_COUNT];
    uint16_t size[F_COUNT];
    const uint32_t* key[KT_COUNT];
    const uint32_t* ypk;          // [keysets][16]
    const uint32_t* row_own;      // [U]
    const uint32_t* row_peer;     // [U]
    const uint32_t* row_st;       // [3][U]
    const uint32_t* peer;         // [U]
    const uint32_t* keyset;       // [U]
    uint8_t* status;              // [U]
    __device__ __forceinline__ uint32_t* p(int f, int u) const { return base + (size_t)off[f] * U + (size_t)u * size[f]; }
    __device__ __forceinline__ const uint32_t* k(int t, uint32_t row) const { return key[t] + (size_t)row * KEY_SIZE_D[t]; }
    __device__ __forceinline__ uint8_t* flags(int u) const { return reinterpret_cast<uint8_t*>(p(F_FLAGS, u)); }
    __device__ __forceinline__ void fail(int u, uint8_t code) const { if (status[u] == 0) status[u] = code; }
};
// FLAGS bytes: 0..2 ZEI ok, 3 peer ciphertext invertible, 6..7 VZEI ok, 8 own ciphertext invertible, 10 range bits, 11..12 MessageB checks ok,
// 13 g_w_vec ok, 14..15 Pedersen ok, 16..17 PDL ok, 18..19 HomoElGamal ok, 20..22 AliceProof challenge ok, 24..27 MessageB DLogProofs ok

// ------------------------------------------------------------------------------ small helpers
__device__ __forceinline__ U256 load_scalar(const uint32_t* p) { return sc_reduce_once(u256_load(p), 0); }

__device__ __forceinline__ void put_point_uncompressed(Sha256& h, const Affine& a) {
    h.put(0x04);
    h.put_fixed(a.x.v, 8);
    h.put_fixed(a.y.v, 8);
}
// `BigInt::from_bytes(P.to_bytes(true))` then chain_bigint: the 33 compressed bytes (first byte 02/03)
__device__ __forceinline__ void put_point_compressed(Sha256& h, const Affine& a) {
    h.put(2 + (a.y.v[0] & 1));
    h.put_fixed(a.x.v, 8);
}
// curv `H::new().chain_points(..).result_scalar()` [R]: 65-byte uncompressed points, digest mod q
static __device__ __noinline__ U256 hash_points_scalar(const Affine* pts, int n) {
    Sha256 h; h.init();
    for (int i = 0; i < n; i++) put_point_uncompressed(h, pts[i]);
    U256 d; h.finish(d.v);
    return sc_reduce_once(d, 0);
}
__device__ __forceinline__ Affine mul_G(const U256& k) { return jac_to_affine(jac_mul_fixed(0, k)); }
__device__ __forceinline__ Affine mul_H(const U256& k) { return jac_to_affine(jac_mul_fixed(1, k)); }
// a*G + b*H and a*G + b*P through the fixed-base tables; the j_ forms stay projective (verifiers compare without inverting)
__device__ __forceinline__ Jac j_lin_GH(const U256& a, const U256& b) { return jac_add(jac_mul_fixed(0, a), jac_mul_fixed(1, b)); }
__device__ __forceinline__ Jac j_lin_GP(const U256& a, const Affine& P, const U256& b) { return jac_add(jac_mul_fixed(0, a), jac_mul(jac_from_affine(P), b)); }
__device__ __forceinline__ Jac j_lin2(const Affine& P, const U256& a, const Affine& Qp, const U256& b) {
    return jac_add(jac_mul(jac_from_affine(P), a), jac_mul(jac_from_affine(Qp), b));
}
__device__ __forceinline__ Jac j_add_aff(const Affine& a, const Affine& b) { return jac_madd(jac_from_affine(a), b); }
__device__ __forceinline__ Affine lin_GH(const U256& a, const U256& b) { return jac_to_affine(j_lin_GH(a, b)); }
__device__ __forceinline__ Affine lin_GP(const U256& a, const Affine& P, const U256& b) { return jac_to_affine(j_lin_GP(a, P, b)); }
__device__ __forceinline__ Affine pt_add_aff(const Affine& a, const Affine& b) { return jac_to_affine(j_add_aff(a, b)); }
// a*P + b*Q
__device__ __forceinline__ Affine lin2(const Affine& P, const U256& a, const Affine& Qp, const U256& b) { return jac_to_affine(j_lin2(P, a, Qp, b)); }
// curv `VerifiableSS::map_share_to_new_params` [R] for two signers of n = 3: lambda_own = x_peer / (x_peer - x_own), tabulated
__device__ __forceinline__ U256 lagrange2(uint32_t own_party, uint32_t peer_party) {
    return u256_load(LAGRANGE2_LIMBS[(own_party % 3) * 3 + (peer_party % 3)]);
}
// curv `DLogProof::prove` [R] (call sites utilities/mta/mod.rs:147-148).  out: pk 16 | T 16 | response 8
static __device__ __noinline__ void dlog_prove(uint32_t* out, const U256& sk, const U256& nonce) {
    Affine pts[3];
    jac_to_affine2(pts[0], pts[2], jac_mul_fixed(0, nonce), jac_mul_fixed(0, sk));        // one shared inversion
    pts[1] = affine_G();
    U256 e = hash_points_scalar(pts, 3);
    U256 resp = sc_sub(nonce, sc_mul(e, sk));
    affine_store(out, pts[2]); affine_store(out + 16, pts[0]); u256_store(out + 32, resp);
}
// curv `DLogProof::verify` [R] (utilities/mta/mod.rs:170-171)
static __device__ __noinline__ bool dlog_verify(const uint32_t* in) {
    Affine pts[3];
    pts[2] = affine_load(in); pts[0] = affine_load(in + 16); pts[1] = affine_G();
    if (pts[2].inf || pts[0].inf || !on_curve(pts[2]) || !on_curve(pts[0])) return false;
    U256 resp = load_scalar(in + 32);
    U256 e = hash_points_scalar(pts, 3);
    return jac_eq_affine(j_lin_GP(resp, pts[2], e), pts[0]);
}
// `HashCommitment::create_commitment_with_user_defined_randomness(from_bytes(compress(P)), blind)` (party_i.rs:577-580)
__device__ __forceinline__ void hash_commit_point(uint32_t* out8, const Affine& P, const uint32_t* blind8) {
    Sha256 h; h.init();
    put_point_compressed(h, P);
    h.put_bigint(blind8, 8);
    h.finish(out8);
}

// commit(Sha256::new().chain_points(pts).result_bigint(); blind): the inner digest re-enters as a minimal-length BigInt
static __device__ __noinline__ void commit_points(uint32_t* out8, const Affine* pts, int n, const uint32_t* blind8) {
    Sha256 h; h.init();
    for (int i = 0; i < n; i++) put_point_uncompressed(h, pts[i]);
    uint32_t d[8];
    h.finish(d);
    Sha256 g; g.init();
    g.put_bigint(d, 8);
    g.put_bigint(blind8, 8);
    g.finish(out8);
}
// e = H(N | N+1 | c | z | u | w); s1 = e*a + alpha; s2 = e*ro + gamma (range_proofs.rs:174-182,87-88)
static __device__ __noinline__ void alice_hash(uint32_t* e8, const uint32_t* N, const uint32_t* c, const uint32_t* z,
                                        const uint32_t* uu, const uint32_t* w) {
    Sha256 h; h.init();
    h.put_bigint(N, 64);
    uint32_t n1[65];
    uint64_t cy = 1;
    for (int i = 0; i < 64; i++) { cy += N[i]; n1[i] = (uint32_t)cy; cy >>= 32; }
    n1[64] = (uint32_t)cy;
    h.put_bigint(n1, 65);
    h.put_bigint(c, 128);
    h.put_bigint(z, 64);
    h.put_bigint(uu, 128);
    h.put_bigint(w, 64);
    h.finish(e8);
}


// ------------------------------------------------------------------------------ round 2
// kzen-paillier CRT decrypt tail [R]: mp = L_p(c^(p-1) mod p^2) * hp mod p, likewise mq,
// m = mp + p * ((mq - mp) * p^-1 mod q)   (call site utilities/mta/mod.rs:165)
static __device__ __noinline__ void decrypt_finish(uint32_t* m64, const Arena& A, uint32_t row, const uint32_t* dp, const uint32_t* dq) {
    uint32_t t[32], lp[32], mp[32], mq[32], scratch[65];
    const uint32_t *p = A.k(KT_P, row), *q = A.k(KT_Q, row);
    // L_p(dp) = (dp - 1) / p, exact: low 1024 bits of (dp - 1) * p^-1 mod 2^1024
    for (int half = 0; half < 2; half++) {
        const uint32_t* d = half ? dq : dp;
        const uint32_t* pr = half ? q : p;
        uint32_t bw = 1;
        for (int i = 0; i < 32; i++) { uint32_t v = d[i]; t[i] = v - bw; bw = (v < bw) ? 1u : 0u; }
        st::mul_low(lp, t, A.k(half ? KT_QINV2 : KT_PINV2, row), 32);
        st::mont_mul(half ? mq : mp, lp, A.k(half ? KT_HQR : KT_HPR, row), pr, st::neg_inv32_st(pr[0]), 32, scratch);
    }
    // diff = (mq - mp) mod q.  Accepted keys have 2^2046 <= pq and p, q < 2^1024 (tecdsa_keys_upload), so q > 2^1022 > p/4:
    // mq - mp > -p > -4q, and at most 4 additions of q make it non-negative
    uint32_t diff[33], mpx[33], qx[33];
    for (int i = 0; i < 32; i++) { diff[i] = mq[i]; mpx[i] = mp[i]; qx[i] = q[i]; }
    diff[32] = 0; mpx[32] = 0; qx[32] = 0;
    st::sub(diff, diff, mpx, 33);
    for (int it = 0; it < 4 && (diff[32] >> 31); it++) st::add(diff, diff, qx, 33);
    while (diff[32] == 0 && st::cmp(diff, q, 32) >= 0) st::sub(diff, diff, qx, 33);
    uint32_t uu[32];
    st::mont_mul(uu, diff, A.k(KT_PINVQR, row), q, st::neg_inv32_st(q[0]), 32, scratch);
    st::mul_add(m64, 64, uu, 32, p, 32, mp, 32);
}

// ------------------------------------------------------------------------------ round 3
// PedersenProof::verify [R] for every signer (sign/rounds.rs:365-378), phase3_reconstruct_delta (party_i.rs:635-640)
static __device__ __noinline__ bool pedersen_verify(const uint32_t* ped, const Affine& com) {
    Affine pts[5];
    pts[0] = affine_G(); pts[1] = affine_H(); pts[2] = com; pts[3] = affine_load(ped + 8); pts[4] = affine_load(ped + 24);
    if (com.inf || !on_curve(com) || !on_curve(pts[3]) || !on_curve(pts[4])) return false;
    U256 e = hash_points_scalar(pts, 5);
    const Jac lhs = j_lin_GH(load_scalar(ped + 40), load_scalar(ped + 48));
    const Jac rhs = jac_add(j_add_aff(pts[3], pts[4]), jac_mul(jac_from_affine(com), e));
    return jac_eq(lhs, rhs);
}

// e = H(G | Q | c | z | u1 | u2 | u3) with points as from_bytes(compressed) (zk_pdl_with_slack/mod.rs:102-110)
static __device__ __noinline__ void pdl_hash(uint32_t* e8, const Affine& Gp, const Affine& Qp, const uint32_t* c, const uint32_t* z,
                                      const Affine& u1, const uint32_t* u2, const uint32_t* u3) {
    Sha256 h; h.init();
    put_point_compressed(h, Gp);
    put_point_compressed(h, Qp);
    h.put_bigint(c, 128);
    h.put_bigint(z, 64);
    put_point_compressed(h, u1);
    h.put_bigint(u2, 128);
    h.put_bigint(u3, 64);
    h.finish(e8);
}

// curv HomoELGamalProof [R] (party_i.rs:778-833)
static __device__ __noinline__ U256 heg_hash(const Affine& T, const Affine& A3, const Affine& Gp, const Affine& D, const Affine& E) {
    Affine pts[7];
    pts[0] = T; pts[1] = A3; pts[2] = Gp; pts[3] = affine_H(); pts[4] = affine_G(); pts[5] = D; pts[6] = E;
    return hash_points_scalar(pts, 7);
}

// ------------------------------------------------------------------------------ round 6 + outputs
static __device__ __noinline__ bool heg_verify(const uint32_t* heg, const Affine& R, const Affine& D, const Affine& E) {
    Affine T = affine_load(heg), A3 = affine_load(heg + 16);
    if (!on_curve(T) || !on_curve(A3) || !on_curve(D) || !on_curve(E)) return false;
    U256 z1 = load_scalar(heg + 32), z2 = load_scalar(heg + 40);
    U256 e = heg_hash(T, A3, R, D, E);
    const Jac l1 = j_lin_GH(z2, z1);                // H*z1 + Y*z2 with Y = G
    const Jac r1 = jac_madd(jac_mul(jac_from_affine(D), e), T);
    const bool ok1 = jac_eq(l1, r1);
    const Jac l2 = jac_mul(jac_from_affine(R), z2);
    const Jac r2 = jac_madd(jac_mul(jac_from_affine(E), e), A3);
    return jac_eq(l2, r2) && ok1;
}
__device__ __forceinline__ void put_point33(Sha256& h, const uint32_t* p16) { put_point_compressed(h, affine_load(p16)); }
__device__ __forceinline__ void put_padded(Sha256& h, const uint32_t* limbs, int have, int want) {
    for (int i = have; i < want; i++) { h.put(0); h.put(0); h.put(0); h.put(0); }
    h.put_fixed(limbs, have);
}


// CRT recombination of an own-key power: x = yp + p^2 * ((yq - yp) * (p^2)^-1 mod q^2)  in [0, N^2)
static __device__ __noinline__ void crt_combine(uint32_t* x128, const Arena& A, uint32_t row, const uint32_t* yp, const uint32_t* yq) {
    const uint32_t *pp = A.k(KT_PP, row), *qq = A.k(KT_QQ, row);
    uint32_t d[65], ypr[65], qx[65], big[129];
    for (int i = 0; i < 64; i++) { d[i] = yq[i]; ypr[i] = yp[i]; qx[i] = qq[i]; }
    d[64] = 0; ypr[64] = 0; qx[64] = 0;
    st::sub(d, d, ypr, 65);
    // p < 4q for every accepted key (see decrypt_finish), so yq - yp > -p^2 > -16 q^2: at most 16 additions
    for (int it = 0; it < 16 && (d[64] >> 31); it++) st::add(d, d, qx, 65);
    uint32_t t[64];
    st::mont_mul(t, d, A.k(KT_PPINVQQR, row), qq, st::neg_inv32_st(qq[0]), 64, big);
    st::mul_add(x128, 128, t, 64, pp, 64, yp, 64);
}

}  // namespace tecdsa
