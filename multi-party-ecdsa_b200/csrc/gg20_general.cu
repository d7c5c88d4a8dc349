// GG20 offline stage for ANY signing set as one batched call (tecdsa_gg20_offline_general_batch): `OfflineStage` Round0..Round6
// of /root/reference/src/protocols/multi_party_ecdsa/gg_2020/state_machine/sign/rounds.rs:68-636 for sessions of T signers of
// key sets of P parties.  The big-integer work is the step functions of the stand-alone L2 entry points (l12_steps.h) on
// flat batches; the bookkeeping between them (indices, Lagrange coefficients, sums, the session stop rule) is
// gg20_general_kernels.cuh, the decommitment check and R are k_gg18_phase4 (gg18.cu).  Everything lives in one Stage, so every
// intermediate is wiped before the call returns.  Same rounds, statuses and stop rule as multi-party-ecdsa_b200/gg20_general.py
// (offline_batch); layouts in include/tecdsa_b200.h and gg20_general_kernels.cuh.
#include "l12_steps.h"
#include "gg20_general_kernels.cuh"

#include <vector>

using namespace tecdsa;

// GG18 phase 4 (gg18_kernels.cuh), defined once in gg18.cu: the decommitment check and R for any number of signers
namespace tecdsa {
namespace gg18 {
__global__ void k_gg18_phase4(int parties, const uint32_t* delta_inv, const uint32_t* b_pk16, const uint32_t* g_gamma16, const uint32_t* blind8,
                              const uint32_t* com8, uint32_t* R16, uint8_t* status, int count);
}  // namespace gg18
}  // namespace tecdsa

extern "C" int tecdsa_gg20_offline_general_batch(tecdsa_ctx* c, const tecdsa_keyset* ks, int signers, size_t n_sessions, int mem, const uint32_t* sessions,
                                                 const tecdsa_offline_general_in* in, const tecdsa_offline_general_out* out) {
    if (!c || !ks || !sessions || !in || !out) return tecdsa_fail(TECDSA_E_ARG, "gg20_offline_general: null argument");
    if (mem != TECDSA_HOST && mem != TECDSA_DEVICE) return tecdsa_fail(TECDSA_E_ARG, "gg20_offline_general: mem must be TECDSA_HOST or TECDSA_DEVICE");
    const int T = signers, P = ks->parties;
    if (T < 2) return tecdsa_fail(TECDSA_E_ARG, "gg20_offline_general: too few signers (TooFewParties)");
    if (T > P) return tecdsa_fail(TECDSA_E_ARG, "gg20_offline_general: more signers than parties");
    if (n_sessions > ((size_t)1 << 24) || n_sessions * (size_t)T * (size_t)P > ((size_t)1 << 26))
        return tecdsa_fail(TECDSA_E_ARG, "gg20_offline_general: too many sessions");
    if (!in->gamma || !in->k || !in->blind || !in->r_k || !in->l || !in->ped_s1 || !in->ped_s2 || !in->heg_s1 || !in->heg_s2 || !in->alice_alpha ||
        !in->alice_beta || !in->alice_gamma || !in->alice_rho || !in->beta_tag_gamma || !in->r_gamma || !in->nonce_gamma_b || !in->nonce_gamma_beta ||
        !in->beta_tag_w || !in->r_w || !in->nonce_w_b || !in->nonce_w_beta || !in->pdl_alpha || !in->pdl_beta || !in->pdl_rho || !in->pdl_gamma ||
        !out->status || !out->R || !out->sigma || !out->T || !out->complete)
        return tecdsa_fail(TECDSA_E_ARG, "gg20_offline_general: null buffer");
    if (n_sessions == 0) return 0;
    CK(cudaSetDevice(c->device));
    // the descriptors are checked on a host copy before anything is touched (sign.rs:87-98: InvalidSl)
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
        if (d[0] >= (uint32_t)ks->n_keysets) return tecdsa_fail(TECDSA_E_ARG, "gg20_offline_general: key set out of range");
        for (int p = 0; p < T; p++) {
            if (d[1 + p] >= (uint32_t)P) return tecdsa_fail(TECDSA_E_ARG, "gg20_offline_general: signer index out of range");
            if (seen >> d[1 + p] & 1) return tecdsa_fail(TECDSA_E_ARG, "gg20_offline_general: repeated signer index (InvalidSl)");
            seen |= (uint64_t)1 << d[1 + p];
        }
    }
    const size_t E = n_sessions * (size_t)T, NP = (size_t)(T - 1) * E, PE = (size_t)P * E;
    const int e = (int)E, np = (int)NP, ns = (int)n_sessions;
    STAGE_PROLOGUE("gg20_offline_general", E);
    const cudaStream_t st = c->stream;
    // ---- inputs (per element, per statement, per pair) and outputs
    const uint32_t* dsess = S.in(sessions, n_sessions * D);
    const uint32_t *gam = S.in(in->gamma, E * 8), *kk = S.in(in->k, E * 8), *blind = S.in(in->blind, E * 8), *rk = S.in(in->r_k, E * 64);
    const uint32_t *ll = S.in(in->l, E * 8), *ps1 = S.in(in->ped_s1, E * 8), *ps2 = S.in(in->ped_s2, E * 8), *hs1 = S.in(in->heg_s1, E * 8),
                   *hs2 = S.in(in->heg_s2, E * 8);
    const uint32_t *aal = S.in(in->alice_alpha, PE * 24), *abe = S.in(in->alice_beta, PE * 64), *aga = S.in(in->alice_gamma, PE * 88),
                   *arh = S.in(in->alice_rho, PE * 72);
    const uint32_t *pal = S.in(in->pdl_alpha, NP * 24), *pbe = S.in(in->pdl_beta, NP * 64), *prh = S.in(in->pdl_rho, NP * 72), *pga = S.in(in->pdl_gamma, NP * 88);
    uint8_t *o_st = S.out(out->status, E), *o_cm = S.out(out->complete, n_sessions);
    uint32_t *o_R = S.out(out->R, E * 16), *o_sg = S.out(out->sigma, E * 8), *o_T = S.out(out->T, E * 16);
    // ---- scratch
    uint32_t *row = S.tmp<uint32_t>(E), *st_row = S.tmp<uint32_t>(PE), *st_elem = S.tmp<uint32_t>(PE);
    uint32_t *pr_me = S.tmp<uint32_t>(2 * NP), *pr_peer = S.tmp<uint32_t>(2 * NP), *pr_row_peer = S.tmp<uint32_t>(2 * NP);
    uint32_t *w = S.tmp<uint32_t>(E * 8), *gw = S.tmp<uint32_t>(E * 16), *g_gamma = S.tmp<uint32_t>(E * 16), *com = S.tmp<uint32_t>(E * 8), *cA = S.tmp<uint32_t>(E * 128);
    uint32_t *er_f = S.tmp<uint32_t>(PE), *a_f = S.tmp<uint32_t>(PE * 8), *r_f = S.tmp<uint32_t>(PE * 64), *c_f = S.tmp<uint32_t>(PE * 128);
    uint32_t *az = S.tmp<uint32_t>(PE * 64), *ae = S.tmp<uint32_t>(PE * 8), *as = S.tmp<uint32_t>(PE * 64), *as1 = S.tmp<uint32_t>(PE * 28), *as2 = S.tmp<uint32_t>(PE * 92);
    uint8_t *pst = S.tmp<uint8_t>(PE), *pair_st = S.tmp<uint8_t>(2 * NP);
    uint32_t *b2 = S.tmp<uint32_t>(2 * NP * 8), *ca2 = S.tmp<uint32_t>(2 * NP * 128), *r2 = S.tmp<uint32_t>(2 * NP * 64), *bt2 = S.tmp<uint32_t>(2 * NP * 64),
             *nb2 = S.tmp<uint32_t>(2 * NP * 8), *nt2 = S.tmp<uint32_t>(2 * NP * 8);
    uint32_t *cb = S.tmp<uint32_t>(2 * NP * 128), *bp = S.tmp<uint32_t>(2 * NP * 40), *btp = S.tmp<uint32_t>(2 * NP * 40), *beta = S.tmp<uint32_t>(2 * NP * 8);
    uint32_t *ak = S.tmp<uint32_t>(2 * NP * 8), *alpha = S.tmp<uint32_t>(2 * NP * 8), *plain = S.tmp<uint32_t>(2 * NP * 64);
    uint8_t *st_b = S.tmp<uint8_t>(2 * NP), *st_a = S.tmp<uint8_t>(2 * NP);
    uint8_t *cand = S.tmp<uint8_t>(E), *status = S.tmp<uint8_t>(E), *stopped = S.tmp<uint8_t>(n_sessions), *ped_st = S.tmp<uint8_t>(E), *st4 = S.tmp<uint8_t>(E);
    uint32_t *delta = S.tmp<uint32_t>(E * 8), *sigma = S.tmp<uint32_t>(E * 8), *Tp = S.tmp<uint32_t>(E * 16), *tproof = S.tmp<uint32_t>(E * 64), *dinv = S.tmp<uint32_t>(E * 8);
    uint32_t *bpk = S.tmp<uint32_t>(E * T * 16), *R = S.tmp<uint32_t>(E * 16), *Rs = S.tmp<uint32_t>(E * 16), *Rd = S.tmp<uint32_t>(E * 16);
    uint32_t *er_p = S.tmp<uint32_t>(NP), *x_p = S.tmp<uint32_t>(NP * 8), *r_p = S.tmp<uint32_t>(NP * 64), *c_p = S.tmp<uint32_t>(NP * 128),
             *Q_p = S.tmp<uint32_t>(NP * 16), *G_p = S.tmp<uint32_t>(NP * 16);
    uint32_t *pz = S.tmp<uint32_t>(NP * 64), *pu1 = S.tmp<uint32_t>(NP * 16), *pu2 = S.tmp<uint32_t>(NP * 128), *pu3 = S.tmp<uint32_t>(NP * 64),
             *pv1 = S.tmp<uint32_t>(NP * 28), *pv2 = S.tmp<uint32_t>(NP * 64), *pv3 = S.tmp<uint32_t>(NP * 92);
    uint8_t *pdl_st = S.tmp<uint8_t>(NP), *heg_st = S.tmp<uint8_t>(E);
    uint32_t *Sp = S.tmp<uint32_t>(E * 16), *heg = S.tmp<uint32_t>(E * 48);
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
    auto gather = [&](uint32_t* dst, const uint32_t* src, int limbs, const uint32_t* idx, size_t count) {
        gen::k_gen_gather<<<grid_for(count), 64, 0, st>>>(dst, src, limbs, idx, (int)count);
        KCHECK();
        return 0;
    };
    auto round_end = [&]() {
        gen::k_gen_round_end<<<grid_for(n_sessions), 64, 0, st>>>(T, cand, status, stopped, ns);
        KCHECK();
        return 0;
    };
    gen::k_gen_index<<<grid_for((size_t)(P > 2 * (T - 1) ? P : 2 * (T - 1)) * E), 64, 0, st>>>(dsess, T, P, e, row, st_row, st_elem, pr_me, pr_peer, pr_row_peer,
                                                                                              (P > 2 * (T - 1) ? P : 2 * (T - 1)) * e);
    KCHECK();
    gen::k_gen_lagrange<<<grid_for(E), 64, 0, st>>>(dsess, T, P, ks->tab[KT_XI], ks->tab[KT_PK], w, gw, e);
    KCHECK();

    // ================= Round 0 (rounds.rs:68-104): g^gamma and its commitment, MessageA with one range proof per keygen party
    RUN(secp_mul_step(c, e, nullptr, gam, g_gamma));
    RUN(hash_commitment_step(c, e, g_gamma, blind, com));
    RUN(mta_encrypt_step(c, S, ks, e, row, kk, rk, cA));
    RUN(gather(er_f, row, 1, st_elem, PE)); RUN(gather(a_f, kk, 8, st_elem, PE)); RUN(gather(r_f, rk, 64, st_elem, PE)); RUN(gather(c_f, cA, 128, st_elem, PE));
    RUN(alice_generate_step(c, S, ks, (int)PE, er_f, st_row, a_f, c_f, r_f, aal, abe, aga, arh, az, ae, as, as1, as2));
    // ================= Round 1 (rounds.rs:122-206): MessageB::b for gamma_i and w_i towards every peer, under the peer's key.
    // The peer's range proofs are verified once per sender and serve all 2 (T - 1) MessageB that answer its MessageA.
    RUN(alice_verify_step(c, S, ks, (int)PE, er_f, st_row, c_f, az, ae, as, as1, as2, pst));
    gen::k_gen_msgb_status<<<grid_for(NP), 64, 0, st>>>(pst, P, T, e, pair_st, np);
    KCHECK();
    RUN(gather(b2, gam, 8, pr_me, NP)); RUN(gather(b2 + NP * 8, w, 8, pr_me, NP)); RUN(gather(ca2, cA, 128, pr_peer, 2 * NP));
    RUN(mta_message_b_step(c, S, ks, 2 * np, pr_row_peer, b2, ca2, r2, bt2, nb2, nt2, 1, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, pair_st,
                           cb, bp, btp, beta, st_b));
    gen::k_gen_round1<<<grid_for(E), 64, 0, st>>>(T, e, st_b, cand, e);
    KCHECK();
    RUN(round_end());
    // ================= Round 2 (rounds.rs:234-317): the peer opens both MessageB; delta_i, sigma_i; T_i and its Pedersen proof
    RUN(gather(ak, kk, 8, pr_peer, 2 * NP));
    RUN(mta_get_alpha_step(c, S, ks, 2 * np, pr_row_peer, ak, cb, bp, btp, alpha, plain, st_a));
    gen::k_gen_round2<<<grid_for(E), 64, 0, st>>>(T, e, st_a, alpha, beta, bp, gw, kk, gam, w, delta, sigma, cand, e);
    KCHECK();
    RUN(pedersen_prove_step(c, e, sigma, ll, ps1, ps2, Tp, tproof));
    RUN(round_end());
    // ================= Round 3 (rounds.rs:347-402): every T_i's Pedersen proof (once per sender), delta^-1
    RUN(pedersen_verify_step(c, e, Tp, tproof, ped_st));
    gen::k_gen_round3<<<grid_for(n_sessions), 64, 0, st>>>(T, delta, ped_st, dinv, cand, ns);
    KCHECK();
    RUN(round_end());
    // ================= Round 4 (rounds.rs:431-498): decommitments and R, R_dash = k_i R, one PDL-with-slack proof per peer
    gen::k_gen_bpk<<<grid_for(E * T), 64, 0, st>>>(T, e, bp, g_gamma, bpk, e * T);
    KCHECK();
    gg18::k_gg18_phase4<<<grid_for(E), 64, 0, st>>>(T, dinv, bpk, g_gamma, blind, com, R, st4, e);
    KCHECK();
    gen::k_gen_round4<<<grid_for(E), 64, 0, st>>>(st4, R, g_gamma, Rs, cand, e);
    KCHECK();
    RUN(secp_mul_step(c, e, Rs, kk, Rd));
    RUN(gather(er_p, row, 1, pr_me, NP)); RUN(gather(x_p, kk, 8, pr_me, NP)); RUN(gather(r_p, rk, 64, pr_me, NP)); RUN(gather(c_p, cA, 128, pr_me, NP));
    RUN(gather(Q_p, Rd, 16, pr_me, NP)); RUN(gather(G_p, Rs, 16, pr_me, NP));
    RUN(pdl_prove_step(c, S, ks, np, er_p, pr_row_peer, x_p, r_p, c_p, Q_p, G_p, pal, pbe, prh, pga, pz, pu1, pu2, pu3, pv1, pv2, pv3));
    RUN(round_end());
    // ================= Round 5 (rounds.rs:525-592): every PDL proof (once each), sum R_dash, S_i and its HomoElGamal proof
    RUN(pdl_verify_step(c, S, ks, np, er_p, pr_row_peer, c_p, Q_p, G_p, pz, pu1, pu2, pu3, pv1, pv2, pv3, pdl_st));
    gen::k_gen_round5<<<grid_for(n_sessions), 64, 0, st>>>(T, e, pdl_st, Rd, cand, ns);
    KCHECK();
    RUN(secp_mul_step(c, e, Rs, sigma, Sp));
    RUN(heg_prove_step(c, e, Rs, Tp, Sp, ll, sigma, hs1, hs2, heg));
    RUN(round_end());
    // ================= Round 6 (rounds.rs:612-636): every HomoElGamal proof (once each), sum S == y
    RUN(heg_verify_step(c, e, Rs, Tp, Sp, heg, heg_st));
    gen::k_gen_round6<<<grid_for(n_sessions), 64, 0, st>>>(T, dsess, heg_st, Sp, ks->ypk, cand, ns);
    KCHECK();
    RUN(round_end());
    gen::k_gen_finish<<<grid_for(E), 64, 0, st>>>(T, status, stopped, R, sigma, Tp, o_st, o_R, o_sg, o_T, o_cm, e);
    KCHECK();
    return S.finish();
}
