// GG18 signing for ANY signing set as one batched call (tecdsa_gg18_signing_batch): phases 1-5, output_signature and verify of
// /root/reference/src/protocols/multi_party_ecdsa/gg_2018/test.rs:163-403 (party_i.rs:385-730) for sessions of T signers of key
// sets of P parties.  The Paillier work is the MtA step functions of the stand-alone L2 entry points (l12_steps.h) with an empty
// statement list; the index tables, Lagrange coefficients and gathers are those of the GG20 general call (gg20_general_kernels.cuh,
// defined in gg20_general.cu); phases 4-5 are the kernels of the GG18 phase entry points (gg18_kernels.cuh, defined in gg18.cu);
// the bookkeeping between them is gg18_signing_kernels.cuh.  Everything lives in one Stage, so every intermediate is wiped before
// the call returns.  Same phases and statuses as multi-party-ecdsa_b200/gg18.py (sign_batch), with the session stop rule of the
// GG20 one-call drivers; layouts in include/tecdsa_b200.h.
#include "l12_steps.h"
#include "gg18_signing_kernels.cuh"

#include <vector>

using namespace tecdsa;

// kernels defined once in other units (gg20_general.cu, gg18.cu)
namespace tecdsa {
namespace gen {
__global__ void k_gen_index(const uint32_t* sess, int T, int P, int E, uint32_t* row, uint32_t* st_row, uint32_t* st_elem, uint32_t* pr_me,
                            uint32_t* pr_peer, uint32_t* pr_row_peer, int threads);
__global__ void k_gen_gather(uint32_t* dst, const uint32_t* src, int limbs, const uint32_t* idx, int count);
__global__ void k_gen_lagrange(const uint32_t* sess, int T, int P, const uint32_t* xi_tab, const uint32_t* pk_tab, uint32_t* w8, uint32_t* gw16, int count);
__global__ void k_gen_bpk(int T, int E, const uint32_t* bp40, const uint32_t* g_gamma16, uint32_t* bpk16, int count);
__global__ void k_gen_round_end(int T, const uint8_t* cand, uint8_t* status, uint8_t* stopped, int sessions);
}  // namespace gen
namespace gg18 {
__global__ void k_gg18_phase4(int parties, const uint32_t* delta_inv, const uint32_t* b_pk16, const uint32_t* g_gamma16, const uint32_t* blind8,
                              const uint32_t* com8, uint32_t* R16, uint8_t* status, int count);
__global__ void k_gg18_local_sig(const uint32_t* msg8, const uint32_t* R16, const uint32_t* k8, const uint32_t* sigma8, uint32_t* s8, int count);
__global__ void k_gg18_phase5a(const uint32_t* R16, const uint32_t* s8, const uint32_t* l8, const uint32_t* rho8, const uint32_t* blind8,
                               const uint32_t* hs1, const uint32_t* hs2, const uint32_t* dnonce, uint32_t* com8, uint32_t* vab48, uint32_t* heg48,
                               uint32_t* dlog40, uint8_t* status, int count);
__global__ void k_gg18_phase5c_senders(const uint32_t* R16, const uint32_t* com8, const uint32_t* vab48, const uint32_t* blind1, const uint32_t* heg48,
                                       const uint32_t* dlog40, uint8_t* verdict, int count);
__global__ void k_gg18_phase5c(int parties, const uint32_t* R16, const uint32_t* y16, const uint32_t* msg8, const uint32_t* rho8, const uint32_t* l8,
                               const uint32_t* blind2, const uint32_t* com8, const uint32_t* vab48, const uint32_t* blind1, const uint32_t* heg48,
                               const uint32_t* dlog40, uint32_t* com2, uint32_t* ut32, uint8_t* status, int count, const uint8_t* sender_ok);
__global__ void k_gg18_phase5d(int parties, const uint32_t* ut32, const uint32_t* blind2, const uint32_t* com2, const uint32_t* vab48, uint8_t* status, int count);
__global__ void k_gg18_output(int parties, const uint32_t* R16, const uint32_t* y16, const uint32_t* msg8, const uint32_t* s8, uint32_t* sig_r,
                              uint32_t* sig_s, uint8_t* recid, uint8_t* status, int count);
}  // namespace gg18
}  // namespace tecdsa

extern "C" int tecdsa_gg18_signing_batch(tecdsa_ctx* c, const tecdsa_keyset* ks, int signers, size_t n_sessions, int mem, const uint32_t* sessions,
                                         const uint32_t* message, const tecdsa_gg18_signing_in* in, const tecdsa_gg18_signing_out* out) {
    if (!c || !ks || !sessions || !message || !in || !out) return tecdsa_fail(TECDSA_E_ARG, "gg18_signing: null argument");
    if (mem != TECDSA_HOST && mem != TECDSA_DEVICE) return tecdsa_fail(TECDSA_E_ARG, "gg18_signing: mem must be TECDSA_HOST or TECDSA_DEVICE");
    const int T = signers, P = ks->parties;
    if (T < 2) return tecdsa_fail(TECDSA_E_ARG, "gg18_signing: too few signers");
    if (T > P) return tecdsa_fail(TECDSA_E_ARG, "gg18_signing: more signers than parties");
    if (n_sessions > ((size_t)1 << 24) || n_sessions * (size_t)T * (size_t)P > ((size_t)1 << 26))
        return tecdsa_fail(TECDSA_E_ARG, "gg18_signing: too many sessions");
    if (!in->k || !in->gamma || !in->blind || !in->r_a || !in->l || !in->rho || !in->blind5 || !in->blind5c || !in->heg_s1 || !in->heg_s2 ||
        !in->dlog_nonce || !in->beta_tag_gamma || !in->r_gamma || !in->beta_tag_w || !in->r_w || !in->nonce_gamma_b || !in->nonce_gamma_beta ||
        !in->nonce_w_b || !in->nonce_w_beta || !out->status || !out->R || !out->sig_r || !out->sig_s || !out->recid || !out->complete)
        return tecdsa_fail(TECDSA_E_ARG, "gg18_signing: null buffer");
    if (n_sessions == 0) return 0;
    CK(cudaSetDevice(c->device));
    // the descriptors are checked on a host copy before anything is touched
    const size_t D = 1 + (size_t)T;
    std::vector<uint32_t> h_sess(n_sessions * D);
    if (mem == TECDSA_HOST) memcpy(h_sess.data(), sessions, h_sess.size() * 4);
    else {
        CK(cudaMemcpyAsync(h_sess.data(), sessions, h_sess.size() * 4, cudaMemcpyDeviceToHost, c->stream));
        CK(cudaStreamSynchronize(c->stream));
    }
    for (size_t s = 0; s < n_sessions; s++) {
        const uint32_t* d = h_sess.data() + s * D;
        uint64_t seen = 0;
        if (d[0] >= (uint32_t)ks->n_keysets) return tecdsa_fail(TECDSA_E_ARG, "gg18_signing: key set out of range");
        for (int p = 0; p < T; p++) {
            if (d[1 + p] >= (uint32_t)P) return tecdsa_fail(TECDSA_E_ARG, "gg18_signing: signer index out of range");
            if (seen >> d[1 + p] & 1) return tecdsa_fail(TECDSA_E_ARG, "gg18_signing: repeated signer index");
            seen |= (uint64_t)1 << d[1 + p];
        }
    }
    const size_t E = n_sessions * (size_t)T, NP = (size_t)(T - 1) * E, PE = (size_t)P * E;
    const int e = (int)E, np = (int)NP, ns = (int)n_sessions;
    const size_t idx_threads = (size_t)(P > 2 * (T - 1) ? P : 2 * (T - 1)) * E;
    STAGE_PROLOGUE("gg18_signing", E);
    const cudaStream_t st = c->stream;
    // ---- inputs and outputs
    const uint32_t *dsess = S.in(sessions, n_sessions * D), *dmsg = S.in(message, n_sessions * 8);
    const uint32_t *kk = S.in(in->k, E * 8), *gam = S.in(in->gamma, E * 8), *blind = S.in(in->blind, E * 8), *ra = S.in(in->r_a, E * 64);
    const uint32_t *ll = S.in(in->l, E * 8), *rho = S.in(in->rho, E * 8), *bl5 = S.in(in->blind5, E * 8), *bl5c = S.in(in->blind5c, E * 8),
                   *hs1 = S.in(in->heg_s1, E * 8), *hs2 = S.in(in->heg_s2, E * 8), *dn = S.in(in->dlog_nonce, E * 8);
    uint8_t *o_st = S.out(out->status, E), *o_rec = S.out(out->recid, n_sessions), *o_cm = S.out(out->complete, n_sessions);
    uint32_t *o_R = S.out(out->R, E * 16), *o_r = S.out(out->sig_r, n_sessions * 8), *o_s = S.out(out->sig_s, n_sessions * 8);
    // ---- scratch
    uint32_t *row = S.tmp<uint32_t>(E), *st_row = S.tmp<uint32_t>(PE), *st_elem = S.tmp<uint32_t>(PE);
    uint32_t *pr_me = S.tmp<uint32_t>(2 * NP), *pr_peer = S.tmp<uint32_t>(2 * NP), *pr_row_peer = S.tmp<uint32_t>(2 * NP);
    uint32_t *w = S.tmp<uint32_t>(E * 8), *gw = S.tmp<uint32_t>(E * 16), *msg = S.tmp<uint32_t>(E * 8), *y = S.tmp<uint32_t>(E * 16);
    uint32_t *g_gamma = S.tmp<uint32_t>(E * 16), *com = S.tmp<uint32_t>(E * 8), *cA = S.tmp<uint32_t>(E * 128);
    uint32_t *b2 = S.tmp<uint32_t>(2 * NP * 8), *ca2 = S.tmp<uint32_t>(2 * NP * 128), *r2 = S.tmp<uint32_t>(2 * NP * 64), *bt2 = S.tmp<uint32_t>(2 * NP * 64),
             *nb2 = S.tmp<uint32_t>(2 * NP * 8), *nt2 = S.tmp<uint32_t>(2 * NP * 8);
    uint32_t *cb = S.tmp<uint32_t>(2 * NP * 128), *bp = S.tmp<uint32_t>(2 * NP * 40), *btp = S.tmp<uint32_t>(2 * NP * 40), *beta = S.tmp<uint32_t>(2 * NP * 8);
    uint32_t *ak = S.tmp<uint32_t>(2 * NP * 8), *alpha = S.tmp<uint32_t>(2 * NP * 8), *plain = S.tmp<uint32_t>(2 * NP * 64);
    uint8_t *st_b = S.tmp<uint8_t>(2 * NP), *st_a = S.tmp<uint8_t>(2 * NP);
    uint8_t *cand = S.tmp<uint8_t>(E), *status = S.tmp<uint8_t>(E), *stopped = S.tmp<uint8_t>(n_sessions), *verdict = S.tmp<uint8_t>(E);
    uint32_t *delta = S.tmp<uint32_t>(E * 8), *sigma = S.tmp<uint32_t>(E * 8), *dinv = S.tmp<uint32_t>(E * 8), *bpk = S.tmp<uint32_t>(E * T * 16),
             *R = S.tmp<uint32_t>(E * 16), *s_i = S.tmp<uint32_t>(E * 8);
    uint32_t *com5 = S.tmp<uint32_t>(E * 8), *vab = S.tmp<uint32_t>(E * 48), *heg = S.tmp<uint32_t>(E * 48), *dlog = S.tmp<uint32_t>(E * 40),
             *com2 = S.tmp<uint32_t>(E * 8), *ut = S.tmp<uint32_t>(E * 32), *sr = S.tmp<uint32_t>(E * 8), *ss = S.tmp<uint32_t>(E * 8);
    uint8_t* rid = S.tmp<uint8_t>(E);
    if (S.err) return S.err;
    // the two MessageB::b of every pair (gamma_i, then w_i) as one batch of 2 NP: the caller's per-pair slabs side by side
    const cudaMemcpyKind kind = mem == TECDSA_HOST ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToDevice;
    const struct { uint32_t* dst; const uint32_t *g, *w; int limbs; } halves[] = {
        {r2, in->r_gamma, in->r_w, 64}, {bt2, in->beta_tag_gamma, in->beta_tag_w, 64}, {nb2, in->nonce_gamma_b, in->nonce_w_b, 8}, {nt2, in->nonce_gamma_beta, in->nonce_w_beta, 8}};
    for (const auto& h : halves) {
        CK(cudaMemcpyAsync(h.dst, h.g, NP * h.limbs * 4, kind, st));
        CK(cudaMemcpyAsync(h.dst + NP * h.limbs, h.w, NP * h.limbs * 4, kind, st));
    }
    CK(cudaMemsetAsync(status, 0, E, st));
    CK(cudaMemsetAsync(stopped, 0, n_sessions, st));
    // phase 5a leaves the messages of a failing element unwritten
    CK(cudaMemsetAsync(com5, 0, E * 8 * 4, st)); CK(cudaMemsetAsync(vab, 0, E * 48 * 4, st));
    CK(cudaMemsetAsync(heg, 0, E * 48 * 4, st)); CK(cudaMemsetAsync(dlog, 0, E * 40 * 4, st));
    auto gather = [&](uint32_t* dst, const uint32_t* src, int limbs, const uint32_t* idx, size_t count) {
        gen::k_gen_gather<<<grid_for(count), 64, 0, st>>>(dst, src, limbs, idx, (int)count);
        KCHECK();
        return 0;
    };
    // the session stop rule at the end of every phase, over the phase's per-element codes
    auto phase_end = [&](const uint8_t* codes) {
        gen::k_gen_round_end<<<grid_for(n_sessions), 64, 0, st>>>(T, codes, status, stopped, ns);
        KCHECK();
        return 0;
    };
    gen::k_gen_index<<<grid_for(idx_threads), 64, 0, st>>>(dsess, T, P, e, row, st_row, st_elem, pr_me, pr_peer, pr_row_peer, (int)idx_threads);
    KCHECK();
    gen::k_gen_lagrange<<<grid_for(E), 64, 0, st>>>(dsess, T, P, ks->tab[KT_XI], ks->tab[KT_PK], w, gw, e);
    KCHECK();
    g18::k_g18_session<<<grid_for(E), 64, 0, st>>>(T, dsess, dmsg, ks->ypk, msg, y, e);
    KCHECK();

    // ================= phase 1 (test.rs:186-198): g^gamma_i and its commitment, MessageA = Enc(k_i) without range proofs
    RUN(secp_mul_step(c, e, nullptr, gam, g_gamma));
    RUN(hash_commitment_step(c, e, g_gamma, blind, com));
    RUN(mta_encrypt_step(c, S, ks, e, row, kk, ra, cA));
    // ================= phase 2 (test.rs:200-290): MessageB::b for gamma_i and w_i towards every peer under the peer's key, then
    // the peer opens both; delta_i and sigma_i
    RUN(gather(b2, gam, 8, pr_me, NP)); RUN(gather(b2 + NP * 8, w, 8, pr_me, NP)); RUN(gather(ca2, cA, 128, pr_peer, 2 * NP));
    RUN(mta_message_b_step(c, S, ks, 2 * np, pr_row_peer, b2, ca2, r2, bt2, nb2, nt2, 0, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr,
                           cb, bp, btp, beta, st_b));
    g18::k_g18_msgb<<<grid_for(E), 64, 0, st>>>(T, e, st_b, cand, e);
    KCHECK();
    RUN(phase_end(cand));
    RUN(gather(ak, kk, 8, pr_peer, 2 * NP));
    RUN(mta_get_alpha_step(c, S, ks, 2 * np, pr_row_peer, ak, cb, bp, btp, alpha, plain, st_a));
    g18::k_g18_phase2<<<grid_for(E), 64, 0, st>>>(T, e, st_a, alpha, beta, kk, gam, w, delta, sigma, cand, e);
    KCHECK();
    RUN(phase_end(cand));
    // ================= phase 3 (test.rs:292-306): delta^-1 of the session sum
    g18::k_g18_phase3<<<grid_for(n_sessions), 64, 0, st>>>(T, delta, dinv, cand, ns);
    KCHECK();
    RUN(phase_end(cand));
    // ================= phase 4 (test.rs:308-327): decommitments, MessageB(gamma) keys, R
    gen::k_gen_bpk<<<grid_for(E * T), 64, 0, st>>>(T, e, bp, g_gamma, bpk, e * T);
    KCHECK();
    gg18::k_gg18_phase4<<<grid_for(E), 64, 0, st>>>(T, dinv, bpk, g_gamma, blind, com, R, cand, e);
    KCHECK();
    RUN(phase_end(cand));
    // ================= phase 5 (test.rs:329-403): s_i, 5a/5b, 5c (each sender's message checked once), 5d, output_signature
    gg18::k_gg18_local_sig<<<grid_for(E), 64, 0, st>>>(msg, R, kk, sigma, s_i, e);
    KCHECK();
    gg18::k_gg18_phase5a<<<grid_for(E), 64, 0, st>>>(R, s_i, ll, rho, bl5, hs1, hs2, dn, com5, vab, heg, dlog, cand, e);
    KCHECK();
    RUN(phase_end(cand));
    gg18::k_gg18_phase5c_senders<<<grid_for(E), 64, 0, st>>>(R, com5, vab, bl5, heg, dlog, verdict, e);
    KCHECK();
    gg18::k_gg18_phase5c<<<grid_for(E), 64, 0, st>>>(T, R, y, msg, rho, ll, bl5c, com5, vab, bl5, heg, dlog, com2, ut, cand, e, verdict);
    KCHECK();
    RUN(phase_end(cand));
    gg18::k_gg18_phase5d<<<grid_for(E), 64, 0, st>>>(T, ut, bl5c, com2, vab, cand, e);
    KCHECK();
    RUN(phase_end(cand));
    gg18::k_gg18_output<<<grid_for(E), 64, 0, st>>>(T, R, y, msg, s_i, sr, ss, rid, cand, e);
    KCHECK();
    RUN(phase_end(cand));
    g18::k_g18_finish<<<grid_for(E), 64, 0, st>>>(T, status, stopped, R, sr, ss, rid, o_st, o_R, o_r, o_s, o_rec, o_cm, e);
    KCHECK();
    return S.finish();
}
