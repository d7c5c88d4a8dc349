// Per-element and per-session kernels of GG18 signing as one call (tecdsa_gg18_signing_batch, gg18_signing.cu): the bookkeeping
// between the MtA steps and the phase kernels of gg18_kernels.cuh that gg18.sign_batch does on the host.  secp256k1 only, one
// thread per element or session.  Element and pair layout of signing_layout.cuh; the two MessageB batches of phase 2 hold two
// halves, h * NP + pair: h = 0 for MessageB(gamma_i), h = 1 for MessageB(w_i) (NP = (T - 1) * E pairs).
// Device code only (no runtime calls), so that tests/host_harness compiles it for the CPU.
#pragma once
#include "signing_layout.cuh"

namespace tecdsa {
namespace g18 {

// per element: the session's message and the public key y of its key set (y_tab = [key sets][16]), the per-element operands of
// phases 5c and output_signature
__global__ void k_g18_session(int T, const uint32_t* sess, const uint32_t* message8, const uint32_t* y_tab, uint32_t* msg8, uint32_t* y16, int count) {
    const int u = blockIdx.x * blockDim.x + threadIdx.x;
    if (u >= count) return;
    const int s = u / T;
    const uint32_t* y = y_tab + (size_t)sess[(size_t)s * (1 + T)] * 16;
    for (int i = 0; i < 8; i++) msg8[(size_t)u * 8 + i] = message8[(size_t)s * 8 + i];
    for (int i = 0; i < 16; i++) y16[(size_t)u * 16 + i] = y[i];
}

// phase 2, MessageB::b (gg_2018/test.rs:203-240): the first failing status of the MessageB element u sent, charged to u as the
// sender; the gamma half first, each half in peer order (the order of gg18.sign_batch)
__global__ void k_g18_msgb(int T, int E, const uint8_t* st_b, uint8_t* cand, int count) {
    const int u = blockIdx.x * blockDim.x + threadIdx.x;
    if (u >= count) return;
    const size_t NP = (size_t)(T - 1) * E;
    uint8_t st = TECDSA_ST_OK;
    for (int h = 0; h < 2; h++)
        for (int j = 0; j < T - 1 && st == TECDSA_ST_OK; j++) st = st_b[h * NP + (size_t)j * E + u];
    cand[u] = st;
}

// phase 2, verify_proofs_get_alpha (test.rs:250-280) and the sums of receiver v: a failed MessageB of either half from any peer
// -> InvalidKey; delta_i = k gamma + sum alpha + sum beta, sigma_i = k w + sum mu + sum nu (party_i.rs:427-445).  st_a / alpha8
// are per pair in the direction b -> v, beta8 per pair as sent.
__global__ void k_g18_phase2(int T, int E, const uint8_t* st_a, const uint32_t* alpha8, const uint32_t* beta8, const uint32_t* k8, const uint32_t* gamma8,
                             const uint32_t* w8, uint32_t* delta8, uint32_t* sigma8, uint8_t* cand, int count) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= count) return;
    const size_t NP = (size_t)(T - 1) * E;
    const U256 k = load_scalar(k8 + (size_t)v * 8);
    U256 delta = sc_mul(k, load_scalar(gamma8 + (size_t)v * 8)), sigma = sc_mul(k, load_scalar(w8 + (size_t)v * 8));
    bool bad = false;
    for (int j = 0; j < T - 1; j++) {
        const size_t in = (size_t)gen::pair_to(T, E, gen::peer_of(T, v, j), v), out = (size_t)j * E + v;
        bad = bad || st_a[in] != TECDSA_ST_OK || st_a[NP + in] != TECDSA_ST_OK;
        delta = sc_add(sc_add(delta, load_scalar(alpha8 + in * 8)), load_scalar(beta8 + out * 8));
        sigma = sc_add(sc_add(sigma, load_scalar(alpha8 + (NP + in) * 8)), load_scalar(beta8 + (NP + out) * 8));
    }
    u256_store(delta8 + (size_t)v * 8, delta);
    u256_store(sigma8 + (size_t)v * 8, sigma);
    cand[v] = bad ? TECDSA_ST_INVALID_KEY : TECDSA_ST_OK;
}

// phase 3 (party_i.rs:447-453) per session: delta = sum delta_i and its inverse for every member; a zero sum (the reference
// panics: "sum of deltas is zero") stops every member with NotInvertible and a zero inverse
__global__ void k_g18_phase3(int T, const uint32_t* delta8, uint32_t* dinv8, uint8_t* cand, int sessions) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= sessions) return;
    const size_t u0 = (size_t)s * T;
    U256 tot = u256_zero();
    for (int p = 0; p < T; p++) tot = sc_add(tot, load_scalar(delta8 + (u0 + p) * 8));
    const bool bad = u256_is_zero(tot);
    const U256 inv = bad ? u256_zero() : sc_inv(tot);
    for (int p = 0; p < T; p++) {
        u256_store(dinv8 + (u0 + p) * 8, inv);
        cand[u0 + p] = bad ? TECDSA_ST_NOT_INVERTIBLE : TECDSA_ST_OK;
    }
}

// outputs of the call: statuses, complete[s], R of every member and the signature of a complete session (zero otherwise); the
// signature is the one signer position 0 derived (k_gg18_output gives every member the same one)
__global__ void k_g18_finish(int T, const uint8_t* status, const uint8_t* stopped, const uint32_t* R16, const uint32_t* r8, const uint32_t* s8,
                             const uint8_t* rid, uint8_t* st_out, uint32_t* R_out, uint32_t* sig_r, uint32_t* sig_s, uint8_t* recid, uint8_t* complete,
                             int count) {
    const int u = blockIdx.x * blockDim.x + threadIdx.x;
    if (u >= count) return;
    const int s = u / T;
    const bool ok = !stopped[s];
    st_out[u] = status[u];
    for (int i = 0; i < 16; i++) R_out[(size_t)u * 16 + i] = ok ? R16[(size_t)u * 16 + i] : 0;
    if (u % T) return;
    complete[s] = ok ? 1 : 0;
    for (int i = 0; i < 8; i++) {
        sig_r[(size_t)s * 8 + i] = ok ? r8[(size_t)u * 8 + i] : 0;
        sig_s[(size_t)s * 8 + i] = ok ? s8[(size_t)u * 8 + i] : 0;
    }
    recid[s] = ok ? rid[u] : 0;
}

}  // namespace g18
}  // namespace tecdsa
