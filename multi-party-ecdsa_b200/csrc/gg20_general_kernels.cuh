// Per-element, per-pair and per-session kernels of the GG20 offline stage for any signing set (tecdsa_gg20_offline_general_batch,
// gg20_general.cu): the bookkeeping between the big-integer steps of sign/rounds.rs:68-636 that the size-generic Python driver does
// on the host.  secp256k1 only, one thread per element, pair or session.
// Element u = s * T + p is signer position p of session s (T signers); pair j * E + u (E = elements, NP = (T - 1) * E pairs) is
// "element u towards its j-th peer", the peer being position ind(p, j) = j < p ? j : j + 1 of the same session.  Round-1 / round-2
// batches hold two halves, h * NP + pair: h = 0 for MessageB(gamma_i), h = 1 for MessageB(w_i).
// sess = [sessions][1 + T]: the key set, then the keygen index - 1 of every signer position.  The index helpers (peer_of,
// pair_to, key_row) are in signing_layout.cuh, shared with the GG18 signing call.
// Device code only (no runtime calls), so that tests/host_harness compiles it for the CPU.
#pragma once
#include "signing_layout.cuh"

namespace tecdsa {
namespace gen {

// Index tables of a call, one thread per entry (threads = max(P, 2 (T - 1)) * E):
//   row[E]            key row of element u;
//   st_row[P * E]     statement x of MessageA's range proofs of element u (t = x * E + u): key row keyset * P + x; st_elem = u;
//   pr_me / pr_peer / pr_row_peer [2 NP]   the sending element, the receiving element and its key row of pair t mod NP.
__global__ void k_gen_index(const uint32_t* sess, int T, int P, int E, uint32_t* row, uint32_t* st_row, uint32_t* st_elem, uint32_t* pr_me,
                            uint32_t* pr_peer, uint32_t* pr_row_peer, int threads) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= threads) return;
    const int NP = (T - 1) * E;
    if (t < E) row[t] = key_row(sess, T, P, t);
    if (t < P * E) {
        const int u = t % E;
        st_row[t] = sess[(size_t)(u / T) * (1 + T)] * (uint32_t)P + (uint32_t)(t / E);
        st_elem[t] = (uint32_t)u;
    }
    if (t < 2 * NP) {
        const int q = t % NP, u = q % E, v = peer_of(T, u, q / E);
        pr_me[t] = (uint32_t)u; pr_peer[t] = (uint32_t)v; pr_row_peer[t] = key_row(sess, T, P, v);
    }
}
// dst[t] = src[idx[t]] for rows of `limbs` limbs
__global__ void k_gen_gather(uint32_t* dst, const uint32_t* src, int limbs, const uint32_t* idx, int count) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= count) return;
    const uint32_t* s = src + (size_t)idx[t] * limbs;
    uint32_t* d = dst + (size_t)t * limbs;
    for (int i = 0; i < limbs; i++) d[i] = s[i];
}

// SignKeys::create / g_w_vec (party_i.rs:527-574): lambda = the Lagrange basis of signer position p at 0 over x_m = l_s[m] + 1
// (curv map_share_to_new_params [R]); w = lambda x_i of its key row; g_w = lambda pk of its key row
__global__ void k_gen_lagrange(const uint32_t* sess, int T, int P, const uint32_t* xi_tab, const uint32_t* pk_tab, uint32_t* w8, uint32_t* gw16, int count) {
    const int u = blockIdx.x * blockDim.x + threadIdx.x;
    if (u >= count) return;
    const uint32_t* d = sess + (size_t)(u / T) * (1 + T) + 1;
    const int p = u % T;
    U256 xj = u256_zero(), num = u256_one(), den = u256_one();
    xj.v[0] = d[p] + 1;
    for (int m = 0; m < T; m++) {
        if (m == p) continue;
        U256 xm = u256_zero();
        xm.v[0] = d[m] + 1;
        num = sc_mul(num, xm);
        den = sc_mul(den, sc_sub(xm, xj));
    }
    const U256 lam = sc_mul(num, sc_inv(den));
    const uint32_t row = key_row(sess, T, P, u);
    u256_store(w8 + (size_t)u * 8, sc_mul(lam, load_scalar(xi_tab + (size_t)row * 8)));
    const Affine pk = affine_load(pk_tab + (size_t)row * 16);
    affine_store(gw16 + (size_t)u * 16, pk.inf ? pk : pt_mul(pk, lam));
}

// MessageB::b's verification of the peer's MessageA (mta/mod.rs:123-131), run once per sender: pst = [P][E] statuses of every
// element's range proofs; pair t (both halves) gets the first failing status of its receiving element's proofs, or OK
__global__ void k_gen_msgb_status(const uint8_t* pst, int P, int T, int E, uint8_t* pair_st, int np) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= np) return;
    const int v = peer_of(T, t % E, t / E);
    uint8_t st = TECDSA_ST_OK;
    for (int x = 0; x < P && st == TECDSA_ST_OK; x++) st = pst[(size_t)x * E + v];
    pair_st[t] = st; pair_st[(size_t)np + t] = st;
}

// round 1 (rounds.rs:122-206): a sender whose MessageB::b failed towards any peer stops with InvalidKey
__global__ void k_gen_round1(int T, int E, const uint8_t* st_b, uint8_t* cand, int count) {
    const int u = blockIdx.x * blockDim.x + threadIdx.x;
    if (u >= count) return;
    const int NP = (T - 1) * E;
    bool bad = false;
    for (int j = 0; j < T - 1; j++) bad = bad || st_b[(size_t)j * E + u] != TECDSA_ST_OK || st_b[(size_t)NP + j * E + u] != TECDSA_ST_OK;
    cand[u] = bad ? TECDSA_ST_INVALID_KEY : TECDSA_ST_OK;
}

// round 2 (rounds.rs:234-317) for receiver v: verify_proofs_get_alpha of both MessageB every peer b sent it, and MessageB(w)'s
// b_proof.pk == g_w_vec[b] (rounds.rs:281) -> InvalidKey; delta_i = k gamma + sum alpha + sum beta, sigma_i = k w + sum mu + sum nu
// (party_i.rs:591-618).  st_a / alpha8 are per pair in the direction b -> v, beta8 / bp40 per pair as sent.
__global__ void k_gen_round2(int T, int E, const uint8_t* st_a, const uint32_t* alpha8, const uint32_t* beta8, const uint32_t* bp40, const uint32_t* gw16,
                             const uint32_t* k8, const uint32_t* gamma8, const uint32_t* w8, uint32_t* delta8, uint32_t* sigma8, uint8_t* cand, int count) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= count) return;
    const size_t NP = (size_t)(T - 1) * E;
    const U256 k = load_scalar(k8 + (size_t)v * 8);
    U256 delta = sc_mul(k, load_scalar(gamma8 + (size_t)v * 8)), sigma = sc_mul(k, load_scalar(w8 + (size_t)v * 8));
    bool bad = false;
    for (int j = 0; j < T - 1; j++) {
        const int b = peer_of(T, v, j);
        const size_t in = (size_t)pair_to(T, E, b, v), out = (size_t)j * E + v;
        bad = bad || st_a[in] != TECDSA_ST_OK || st_a[NP + in] != TECDSA_ST_OK || !eq16(bp40 + (NP + in) * 40, gw16 + (size_t)b * 16);
        delta = sc_add(sc_add(delta, load_scalar(alpha8 + in * 8)), load_scalar(beta8 + out * 8));
        sigma = sc_add(sc_add(sigma, load_scalar(alpha8 + (NP + in) * 8)), load_scalar(beta8 + (NP + out) * 8));
    }
    u256_store(delta8 + (size_t)v * 8, delta);
    u256_store(sigma8 + (size_t)v * 8, sigma);
    cand[v] = bad ? TECDSA_ST_INVALID_KEY : TECDSA_ST_OK;
}

// round 3 (rounds.rs:347-402) per session: delta = sum delta_i and its inverse (party_i.rs:635-640) for every member; a failed
// Pedersen proof of any member (verified once per sender) or delta = 0 stops every member with the proof error
__global__ void k_gen_round3(int T, const uint32_t* delta8, const uint8_t* ped_st, uint32_t* dinv8, uint8_t* cand, int sessions) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= sessions) return;
    const size_t u0 = (size_t)s * T;
    U256 tot = u256_zero();
    bool bad = false;
    for (int p = 0; p < T; p++) {
        tot = sc_add(tot, load_scalar(delta8 + (u0 + p) * 8));
        bad = bad || ped_st[u0 + p] != TECDSA_ST_OK;
    }
    bad = bad || u256_is_zero(tot);
    const U256 inv = bad ? u256_zero() : sc_inv(tot);
    for (int p = 0; p < T; p++) {
        u256_store(dinv8 + (u0 + p) * 8, inv);
        cand[u0 + p] = bad ? TECDSA_ST_PROOF : TECDSA_ST_OK;
    }
}

// round 4 (rounds.rs:431-498): the b_proof_pk table of k_gg18_phase4, thread (u, j): the public key of MessageB(gamma) that
// signer position j sent element u, and u's own g^gamma at its own position
__global__ void k_gen_bpk(int T, int E, const uint32_t* bp40, const uint32_t* g_gamma16, uint32_t* bpk16, int count) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= count) return;
    const int u = t / T, b = u - u % T + t % T;
    const uint32_t* src = b == u ? g_gamma16 + (size_t)u * 16 : bp40 + (size_t)pair_to(T, E, b, u) * 40;
    uint32_t* d = bpk16 + (size_t)t * 16;
    for (int i = 0; i < 16; i++) d[i] = src[i];
}
// after k_gg18_phase4: a failed decommitment check stops the element with the commitment error; Rs = R, or g^gamma where R is the
// identity (only in a session that has stopped: its later rounds then still run on curve points)
__global__ void k_gen_round4(const uint8_t* st4, const uint32_t* R16, const uint32_t* g_gamma16, uint32_t* Rs16, uint8_t* cand, int count) {
    const int u = blockIdx.x * blockDim.x + threadIdx.x;
    if (u >= count) return;
    const Affine R = affine_load(R16 + (size_t)u * 16);
    affine_store(Rs16 + (size_t)u * 16, R.inf ? affine_load(g_gamma16 + (size_t)u * 16) : R);
    cand[u] = st4[u] != TECDSA_ST_OK ? TECDSA_ST_COMMITMENT : TECDSA_ST_OK;
}

// round 5 (rounds.rs:525-592) per session: every member's PDL proofs (each verified once) -> PDL error for all; else
// sum R_dash != G (party_i.rs:768-776) -> the phase-5 error for all
__global__ void k_gen_round5(int T, int E, const uint8_t* pdl_st, const uint32_t* Rdash16, uint8_t* cand, int sessions) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= sessions) return;
    const size_t u0 = (size_t)s * T;
    bool bad = false;
    Jac acc = jac_identity();
    for (int p = 0; p < T; p++) {
        for (int j = 0; j < T - 1; j++) bad = bad || pdl_st[(size_t)j * E + u0 + p] != TECDSA_ST_OK;
        acc = jac_madd(acc, affine_load(Rdash16 + (u0 + p) * 16));
    }
    const uint8_t st = bad ? TECDSA_ST_PDL_VERIFY : !jac_eq_affine(acc, affine_G()) ? TECDSA_ST_PHASE5_BAD_SUM : TECDSA_ST_OK;
    for (int p = 0; p < T; p++) cand[u0 + p] = st;
}

// round 6 (rounds.rs:612-636) per session: every member's HomoELGamal proof (each verified once) and sum S == y_sum_s of the key set
// (party_i.rs:801-848), else the phase-6 error for all
__global__ void k_gen_round6(int T, const uint32_t* sess, const uint8_t* heg_st, const uint32_t* S16, const uint32_t* y_tab, uint8_t* cand, int sessions) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= sessions) return;
    const size_t u0 = (size_t)s * T;
    bool bad = false;
    Jac acc = jac_identity();
    for (int p = 0; p < T; p++) {
        bad = bad || heg_st[u0 + p] != TECDSA_ST_OK;
        acc = jac_madd(acc, affine_load(S16 + (u0 + p) * 16));
    }
    bad = bad || !jac_eq_affine(acc, affine_load(y_tab + (size_t)sess[(size_t)s * (1 + T)] * 16));
    for (int p = 0; p < T; p++) cand[u0 + p] = bad ? TECDSA_ST_PHASE6 : TECDSA_ST_OK;
}

// the session stop rule, at the end of every round: a member records this round's error only while its session runs, and the
// session stops when any member has an error
__global__ void k_gen_round_end(int T, const uint8_t* cand, uint8_t* status, uint8_t* stopped, int sessions) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= sessions || stopped[s]) return;
    const size_t u0 = (size_t)s * T;
    bool any = false;
    for (int p = 0; p < T; p++) {
        if (status[u0 + p] == TECDSA_ST_OK) status[u0 + p] = cand[u0 + p];
        any = any || status[u0 + p] != TECDSA_ST_OK;
    }
    stopped[s] = any ? 1 : 0;
}

// outputs of the call: statuses, complete[s], and R, sigma_i, T_i of every member of a complete session (zero otherwise)
__global__ void k_gen_finish(int T, const uint8_t* status, const uint8_t* stopped, const uint32_t* R16, const uint32_t* sigma8, const uint32_t* T16,
                             uint8_t* st_out, uint32_t* R_out, uint32_t* sigma_out, uint32_t* T_out, uint8_t* complete, int count) {
    const int u = blockIdx.x * blockDim.x + threadIdx.x;
    if (u >= count) return;
    const bool ok = !stopped[u / T];
    st_out[u] = status[u];
    if (u % T == 0) complete[u / T] = ok ? 1 : 0;
    for (int i = 0; i < 16; i++) R_out[(size_t)u * 16 + i] = ok ? R16[(size_t)u * 16 + i] : 0;
    for (int i = 0; i < 8; i++) sigma_out[(size_t)u * 8 + i] = ok ? sigma8[(size_t)u * 8 + i] : 0;
    for (int i = 0; i < 16; i++) T_out[(size_t)u * 16 + i] = ok ? T16[(size_t)u * 16 + i] : 0;
}

}  // namespace gen
}  // namespace tecdsa
