// Per-element, per-pair and per-group kernels of the GG20 key generation (tecdsa_gg20_keygen_batch, keygen.cu): the group-level
// steps between the big-integer proofs of gg_2020/party_i.rs:260-438, secp256k1 and SHA-256 only, one thread per element, pair or
// coefficient.  Element e = g * n + (i - 1) is party i of group g; pair p = e * n + s is "receiver e checks sender g * n + s".
// Device code only (no runtime calls), so that tests/host_harness compiles it for the CPU.
#pragma once
#include "gg20_glue.cuh"

namespace tecdsa {
namespace kg {

__device__ __forceinline__ int bit_length64(const uint32_t* x) {
    int top = 63;
    while (top > 0 && x[top] == 0) top--;
    return x[top] ? top * 32 + (32 - __clz(x[top])) : 0;
}
__device__ __forceinline__ bool limbs_eq(const uint32_t* a, const uint32_t* b, int k) {
    uint32_t x = 0;
    for (int j = 0; j < k; j++) x |= a[j] ^ b[j];
    return x == 0;
}
// curv `VerifiableSS::get_point_commitment(index)` [R]: sum_j index^j * C_j by Horner from the top.  ok = false for a commitment
// that is not on the curve (the identity, all-zero, is accepted as curv's zero point).
__device__ __forceinline__ Jac point_commitment(const uint32_t* C, int n_comm, uint32_t index, bool& ok) {
    U256 idx = u256_zero();
    idx.v[0] = index;
    ok = n_comm > 0;
    Jac acc = jac_identity();
    for (int j = n_comm - 1; j >= 0 && ok; j--) {
        Affine cj = affine_load(C + (size_t)j * 16);
        if (!cj.inf && !on_curve(cj)) { ok = false; break; }
        if (j != n_comm - 1) acc = jac_mul(acc, idx);
        acc = jac_add(acc, jac_from_affine(cj));
    }
    return acc;
}
// curv `VerifiableSS::validate_share(&share, index)` [R] (party_i.rs:337-339): share * G == get_point_commitment(index)
__device__ __forceinline__ bool vss_share_ok(const uint32_t* C, int n_comm, const uint32_t* share, uint32_t index) {
    bool ok;
    const Jac acc = point_commitment(C, n_comm, index, ok);
    const Affine lhs = mul_G(sc_from_limbs(share, 8));
    return ok && affine_eq(lhs, jac_to_affine(acc));
}
// the decommitment (y_i, blind) reopens com (party_i.rs:277-281); the digest is consumed where it is made (DESIGN.md, last rule)
static __device__ __noinline__ bool commit_reopens(const uint32_t* y16, const uint32_t* blind8, const uint32_t* com8) {
    uint32_t d[8];
    hash_commit_point(d, affine_load(y16), blind8);
    return limbs_eq(d, com8, 8);
}

// Round 1 (party_i.rs:219-258): com = HashCommitment(compressed y_i; blind) with y_i = u_i * G = the party's commitment 0
__global__ void k_kg_commit(const uint32_t* comm, int t1, const uint32_t* blind8, uint32_t* com8, int count) {
    int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= count) return;
    hash_commit_point(com8 + (size_t)e * 8, affine_load(comm + (size_t)e * t1 * 16), blind8 + (size_t)e * 8);
}

// Round 2, once per sender (party_i.rs:272-305): the commitment reopens, NiCorrectKeyProof verifies (st_ck), N and N~ have
// 2047..2048 bits, both CompositeDLogProofs verify (st_cd[e], st_cd[count + e]).  y16 = [count] rows of y_stride limbs.
__global__ void k_kg_round2(const uint32_t* y16, int y_stride, const uint32_t* blind8, const uint32_t* com8, const uint8_t* st_ck, const uint32_t* n64,
                            const uint32_t* nt64, const uint8_t* st_cd, uint8_t* ok2, int count) {
    int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= count) return;
    const int bn = bit_length64(n64 + (size_t)e * 64), bt = bit_length64(nt64 + (size_t)e * 64);
    const bool ok = commit_reopens(y16 + (size_t)e * y_stride, blind8 + (size_t)e * 8, com8 + (size_t)e * 8) && st_ck[e] == TECDSA_ST_OK &&
                    bn >= 2047 && bn <= 2048 && bt >= 2047 && bt <= 2048 && st_cd[e] == TECDSA_ST_OK && st_cd[count + e] == TECDSA_ST_OK;
    ok2[e] = ok ? 1 : 0;
}

// Round 3, one thread per (receiver, sender) pair of a group (party_i.rs:334-349): the sender's share for this receiver validates
// against the sender's commitments, and the sender's commitment 0 equals its decommitted y.  comm = [E][t1][16],
// shares = [E][n][8] (row s * n + r = sender s's share for party r + 1), y16 as in k_kg_round2.
__global__ void k_kg_validate_pairs(const uint32_t* comm, int t1, const uint32_t* y16, int y_stride, const uint32_t* shares, int n, uint8_t* pair_ok,
                                    int pairs) {
    int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= pairs) return;
    const int e = p / n, s = p % n;
    const int r = e % n, snd = e - r + s;
    const uint32_t* C = comm + (size_t)snd * t1 * 16;
    const bool ok = vss_share_ok(C, t1, shares + ((size_t)snd * n + r) * 8, (uint32_t)(r + 1)) && limbs_eq(C, y16 + (size_t)snd * y_stride, 16);
    pair_ok[p] = ok ? 1 : 0;
}

// Round 3 (party_i.rs:351-362): x_i = sum over the group's senders of their shares for party i, mod q
__global__ void k_kg_xi(const uint32_t* shares, int n, uint32_t* x8, int count) {
    int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= count) return;
    const int r = e % n, g0 = e - r;
    U256 acc = u256_zero();
    for (int s = 0; s < n; s++) acc = sc_add(acc, sc_from_limbs(shares + ((size_t)(g0 + s) * n + r) * 8, 8));
    u256_store(x8 + (size_t)e * 8, acc);
}

// DLogProof::prove(&x_i) (party_i.rs:364) with the sampled nonce explicit
__global__ void k_kg_dlog_prove(const uint32_t* x8, const uint32_t* nonce8, uint32_t* proof40, int count) {
    int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= count) return;
    dlog_prove(proof40 + (size_t)e * 40, sc_from_limbs(x8 + (size_t)e * 8, 8), sc_from_limbs(nonce8 + (size_t)e * 8, 8));
}

// `get_commitments_to_xi` first half (party_i.rs:369-383): the global commitment k of group g = sum over its parties of C_{j,k};
// thread (g, k).  gcomm = [groups][t1][16].  Commitment 0 is also y_sum_s: y_j is party j's commitment 0 (keygen/rounds.rs:278-279).
__global__ void k_kg_global_commitments(const uint32_t* comm, int t1, int n, uint32_t* gcomm, int groups) {
    int id = blockIdx.x * blockDim.x + threadIdx.x;
    if (id >= groups * t1) return;
    const int g = id / t1, k = id % t1;
    Jac acc = jac_identity();
    for (int j = 0; j < n; j++) acc = jac_add(acc, jac_from_affine(affine_load(comm + ((size_t)(g * n + j) * t1 + k) * 16)));
    affine_store(gcomm + (size_t)id * 16, jac_to_affine(acc));
}

// Round 4, once per sender (party_i.rs:405-438): DLogProof::verify and pk == get_point_commitment(i) of the group's global
// commitments (Horner, compared projectively)
__global__ void k_kg_round4(const uint32_t* gcomm, int t1, int n, const uint32_t* proof40, uint8_t* ok4, int count) {
    int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= count) return;
    const uint32_t* pf = proof40 + (size_t)e * 40;
    bool ok;
    const Jac xi = point_commitment(gcomm + (size_t)(e / n) * t1 * 16, t1, (uint32_t)(e % n + 1), ok);
    ok4[e] = (ok && dlog_verify(pf) && jac_eq_affine(xi, affine_load(pf))) ? 1 : 0;
}

// Status, bad actors and completion per element.  A group stops at the first round in which one of its members failed:
//   round 0  an xhi with no inverse mod phi(N~) (st_nt): that element NOT_INVERTIBLE, mask 0;
//   round 2  any sender failed (ok2): every element INVALID_KEY with the mask of all failing senders;
//   round 3  any pair failed (pair_ok): each receiver with a failing sender INVALID_SS with its own mask;
//   round 4  any sender failed (ok4): every element PROOF with the mask of all failing senders.
// Bit j of a mask = party j + 1.  complete[g] = 1 iff no round failed; then pk[g][i] = the DLog proof's pk and y[g] = the global
// commitment 0, else those and the element's LocalKey rows (x8, vss, n64, dlog_st) are zeroed.
__global__ void k_kg_finish(int n, int t1, const uint8_t* st_nt, const uint8_t* ok2, const uint8_t* pair_ok, const uint8_t* ok4, const uint32_t* proof40,
                            const uint32_t* gcomm, uint8_t* status, uint64_t* bad, uint8_t* complete, uint32_t* pk16, uint32_t* y16, uint32_t* x8,
                            uint32_t* vss, uint32_t* n64, uint32_t* dlog_st, int count) {
    int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= count) return;
    const int i = e % n, g0 = e - i;
    bool r0 = true, r3 = true;
    uint64_t m2 = 0, m3 = 0, m4 = 0;
    for (int j = 0; j < n; j++) {
        r0 = r0 && st_nt[g0 + j] == TECDSA_ST_OK;
        if (!ok2[g0 + j]) m2 |= 1ull << j;
        if (!ok4[g0 + j]) m4 |= 1ull << j;
        if (!pair_ok[(size_t)e * n + j]) m3 |= 1ull << j;
        for (int s = 0; s < n; s++) r3 = r3 && pair_ok[(size_t)(g0 + j) * n + s];
    }
    uint8_t st = TECDSA_ST_OK;
    uint64_t mask = 0;
    if (!r0) st = st_nt[e];
    else if (m2) { st = TECDSA_ST_INVALID_KEY; mask = m2; }
    else if (!r3) { st = m3 ? TECDSA_ST_INVALID_SS : TECDSA_ST_OK; mask = m3; }
    else if (m4) { st = TECDSA_ST_PROOF; mask = m4; }
    const bool done = r0 && !m2 && r3 && !m4;
    status[e] = st;
    bad[e] = mask;
    const int g = e / n;
    for (int k = 0; k < 16; k++) pk16[(size_t)e * 16 + k] = done ? proof40[(size_t)e * 40 + k] : 0u;
    if (i == 0) {
        complete[g] = done ? 1 : 0;
        for (int k = 0; k < 16; k++) y16[(size_t)g * 16 + k] = done ? gcomm[(size_t)g * t1 * 16 + k] : 0u;
    }
    if (!done) {
        for (int k = 0; k < 8; k++) x8[(size_t)e * 8 + k] = 0;
        for (int k = 0; k < t1 * 16; k++) vss[(size_t)e * t1 * 16 + k] = 0;
        for (int k = 0; k < 64; k++) n64[(size_t)e * 64 + k] = 0;
        for (int k = 0; k < 3 * 64; k++) dlog_st[(size_t)e * 3 * 64 + k] = 0;
    }
}

}  // namespace kg
}  // namespace tecdsa
