// The kernels of the batched GG20 offline stage, one per step between the big-integer job launches (see gg20.cu for the order):
// EC arithmetic, Fiat-Shamir hashing, plain-integer responses, Paillier CRT recombination, the sigma proofs of curv and the
// per-round checks, built from the device functions of gg20_glue.cuh.  Included by gg20.cu (and the host test harness) only —
// the other translation units need the device functions, not these kernels.
#pragma once
#include "gg20_glue.cuh"

namespace tecdsa {

// ------------------------------------------------------------------------------ round 0
// SignKeys::create + phase1_broadcast (party_i.rs:546-589) and the plain factors of MessageA::a
// (utilities/mta/mod.rs:68-75, range_proofs.rs:53).
static __global__ void gg20_r0_pre(Arena A) {
    int u = blockIdx.x * blockDim.x + threadIdx.x;
    if (u >= A.U) return;
    const uint32_t* rnd = A.p(F_RND, u);
    const uint32_t row = A.row_own[u];
    U256 lam = lagrange2(row % 3, A.row_peer[u] % 3);
    U256 w = sc_mul(lam, load_scalar(A.k(KT_XI, row)));
    u256_store(A.p(F_W, u), w);
    Affine gg = mul_G(load_scalar(rnd + RND_GAMMA));
    affine_store(A.p(F_GG, u), gg);
    hash_commit_point(A.p(F_COM, u), gg, rnd + RND_BLIND);
    const uint32_t* N = A.k(KT_N, row);
    uint32_t one = 1;
    st::mul_add(A.p(F_MK, u), 128, rnd + RND_K, 8, N, 64, &one, 1);
    for (int x = 0; x < 3; x++)
        st::mul_add(A.p(F_ALIN0 + x, u), 128, rnd + RND_AL + x * RND_AL_STRIDE + RND_AL_ALPHA, 24, N, 64, &one, 1);
}

static __global__ void gg20_r0_mid(Arena A) {
    int u = blockIdx.x * blockDim.x + threadIdx.x;
    if (u >= A.U) return;
    const uint32_t* rnd = A.p(F_RND, u);
    const uint32_t* N = A.k(KT_N, A.row_own[u]);
    for (int x = 0; x < 3; x++) {
        const uint32_t* al = rnd + RND_AL + x * RND_AL_STRIDE;
        uint32_t* e = A.p(F_E0 + x, u);
        alice_hash(e, N, A.p(F_CK, u), A.p(F_Z0 + x, u), A.p(F_U0 + x, u), A.p(F_WP0 + x, u));
        st::mul_add(A.p(F_S10 + x, u), 28, e, 8, rnd + RND_K, 8, al + RND_AL_ALPHA, 24);
        st::mul_add(A.p(F_S20 + x, u), 92, e, 8, al + RND_AL_RHO, 72, al + RND_AL_GAMMA, 88);
    }
}

// ------------------------------------------------------------------------------ round 1
// AliceProof::verify prologue for the peer's proofs (range_proofs.rs:118,134) and the plain
// factor of Paillier encrypt inside MessageB::b (utilities/mta/mod.rs:133).
static __global__ void gg20_r1_pre(Arena A) {
    int u = blockIdx.x * blockDim.x + threadIdx.x;
    if (u >= A.U) return;
    const int pu = A.peer[u];
    const uint32_t* rnd = A.p(F_RND, u);
    const uint32_t* Np = A.k(KT_N, A.row_peer[u]);
    uint32_t one = 1;
    uint8_t* fl = A.flags(u);
    uint8_t rng = 0;
    for (int x = 0; x < 3; x++) {
        const uint32_t* s1 = A.p(F_S10 + x, pu);
        if (st::cmp2(s1, 28, Q3_LIMBS, 24) > 0) rng |= (1u << x);
        st::mul_add(A.p(F_GS10 + x, u), 128, s1, 28, Np, 64, &one, 1);
    }
    fl[10] = rng;
    st::mul_add(A.p(F_LBG, u), 128, rnd + RND_BT_G, 64, Np, 64, &one, 1);
    st::mul_add(A.p(F_LBW, u), 128, rnd + RND_BT_W, 64, Np, 64, &one, 1);
}

// end of AliceProof::verify (range_proofs.rs:143-153): one thread per (unit, statement)
static __global__ void gg20_r1_post_hash(Arena A) {
    int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= A.U * 3) return;
    const int u = t / 3, x = t % 3, pu = A.peer[u];
    uint32_t* e = A.p(F_DBG, u) + 8 * x;          // recomputed challenge (kept in the arena)
    alice_hash(e, A.k(KT_N, A.row_peer[u]), A.p(F_CK, pu), A.p(F_Z0 + x, pu), A.p(F_UV0 + x, u), A.p(F_WV0 + x, u));
    A.flags(u)[20 + x] = st::cmp(e, A.p(F_E0 + x, pu), 8) == 0;
}

// rest of MessageB::b (mta/mod.rs:132,146-148): one thread per (unit, DLogProof)
static __global__ void gg20_r1_post_dlog(Arena A) {
    int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= A.U * 4) return;
    const int u = t >> 2, j = t & 3;
    const uint32_t* rnd = A.p(F_RND, u);
    U256 sk;
    if (j == 0) sk = load_scalar(rnd + RND_GAMMA);
    else if (j == 2) sk = u256_load(A.p(F_W, u));
    else {
        sk = sc_from_limbs(rnd + (j == 1 ? RND_BT_G : RND_BT_W), 64);
        u256_store(A.p(j == 1 ? F_BTG_FE : F_BTW_FE, u), sk);
        u256_store(A.p(j == 1 ? F_BETA_G : F_NU, u), sc_neg(sk));
    }
    const int nonce_off = j == 0 ? RND_NB_G : j == 1 ? RND_NBT_G : j == 2 ? RND_NB_W : RND_NBT_W;
    dlog_prove(A.p(F_DL0 + j, u), sk, load_scalar(rnd + nonce_off));
}

// MessageB::verify_proofs_get_alpha (mta/mod.rs:160-179): threads (unit, 0) and (unit, 1) handle the gamma and the
// w message (Paillier CRT tail, G*alpha == B*k + B'); threads (unit, 2..5) the four DLogProofs; thread (unit, 6) the g_w_vec assert
// (sign/rounds.rs:281)
static __global__ void gg20_r2_check(Arena A) {
    int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= A.U * 7) return;
    const int job = t / A.U, u = t % A.U, pu = A.peer[u];     // task-major: the threads of a warp run the same kind of check
    const uint32_t row = A.row_own[u], prow = A.row_peer[u];
    if (job == 6) {
        const Jac gw = jac_mul(jac_from_affine(affine_load(A.k(KT_PK, prow))), lagrange2(prow % 3, row % 3));
        A.flags(u)[13] = jac_eq_affine(gw, affine_load(A.p(F_DL2, pu)));
        return;
    }
    const int m = job & 1;
    const uint32_t* bp = A.p(m ? F_DL2 : F_DL0, pu);
    const uint32_t* btp = A.p(m ? F_DL3 : F_DL1, pu);
    if (job >= 2) {                                  // the two DLogProofs of each MessageB, one thread each
        const bool second = job >= 4;
        A.flags(u)[24 + 2 * m + (second ? 1 : 0)] = dlog_verify(second ? btp : bp);
        return;
    }
    // the plaintext goes to the arena (it is also part of the reference's return value, mta/mod.rs:175)
    uint32_t* plain = A.p(m ? F_APLW : F_APLG, u);
    decrypt_finish(plain, A, row, A.p(m ? F_DPW : F_DPG, u), A.p(m ? F_DQW : F_DQG, u));
    U256 alpha = sc_from_limbs(plain, 64);
    u256_store(A.p(m ? F_MU : F_ALPHA, u), alpha);
    const U256 k = load_scalar(A.p(F_RND, u) + RND_K);
    const Jac ba_btag = jac_madd(jac_mul(jac_from_affine(affine_load(bp)), k), affine_load(btp));
    A.flags(u)[11 + m] = jac_eq(ba_btag, jac_mul_fixed(0, alpha));
}

// phase2_delta_i / phase2_sigma_i (party_i.rs:591-618), phase3_compute_t_i + PedersenProof::prove [R] (party_i.rs:620-634)
static __global__ void gg20_r2_finish(Arena A) {
    int u = blockIdx.x * blockDim.x + threadIdx.x;
    if (u >= A.U) return;
    const uint32_t* rnd = A.p(F_RND, u);
    const uint8_t* fl = A.flags(u);
    bool ok1 = fl[10] == 0;
    for (int x = 0; x < 3; x++) ok1 = ok1 && fl[x] && fl[3] && fl[20 + x];      // fl[3]: the peer's ciphertext is invertible mod N^2
    if (!ok1) A.fail(u, TECDSA_ST_INVALID_KEY);                    // MessageB::b -> Err(InvalidKey) (mta/mod.rs:123-131)
    if (!(fl[11] && fl[12] && fl[13] && fl[24] && fl[25] && fl[26] && fl[27])) A.fail(u, TECDSA_ST_INVALID_KEY);
    const U256 k = load_scalar(rnd + RND_K), gamma = load_scalar(rnd + RND_GAMMA), w = u256_load(A.p(F_W, u));
    U256 delta = sc_add(sc_add(sc_mul(k, gamma), u256_load(A.p(F_ALPHA, u))), u256_load(A.p(F_BETA_G, u)));
    U256 sigma = sc_add(sc_add(sc_mul(k, w), u256_load(A.p(F_MU, u))), u256_load(A.p(F_NU, u)));
    u256_store(A.p(F_DELTA, u), delta); u256_store(A.p(F_SIGMA, u), sigma);
    const U256 l = load_scalar(rnd + RND_L);
    const U256 s1 = load_scalar(rnd + RND_PED_S1), s2 = load_scalar(rnd + RND_PED_S2);
    Affine pts[5];
    jac_to_affine3(pts[2], pts[3], pts[4], j_lin_GH(sigma, l), jac_mul_fixed(0, s1), jac_mul_fixed(1, s2));     // T, a1, a2: one inversion
    const Affine T = pts[2];
    affine_store(A.p(F_T, u), T);
    pts[0] = affine_G(); pts[1] = affine_H();
    U256 e = hash_points_scalar(pts, 5);
    uint32_t* ped = A.p(F_PED, u);
    u256_store(ped, e); affine_store(ped + 8, pts[3]); affine_store(ped + 24, pts[4]);
    u256_store(ped + 40, sc_add(s1, sc_mul(e, sigma))); u256_store(ped + 48, sc_add(s2, sc_mul(e, l)));
}

// PedersenProof::verify of the unit's own proof.  Both signers of a session check every proof of the session on the same inputs
// (no input comes from the verifier's side), so each proof is checked once, on its prover's unit, and the peer's finish kernel
// reads that verdict (declared shortcut 10, DESIGN.md section 4).  The same holds for the PDL and HomoElGamal checks below.
static __global__ void gg20_r3_check(Arena A) {
    int u = blockIdx.x * blockDim.x + threadIdx.x;
    if (u >= A.U) return;
    A.flags(u)[14] = pedersen_verify(A.p(F_PED, u), affine_load(A.p(F_T, u)));
}

static __global__ void gg20_r3_finish(Arena A) {
    int u = blockIdx.x * blockDim.x + threadIdx.x;
    if (u >= A.U) return;
    const int pu = A.peer[u];
    if (!(A.flags(u)[14] && A.flags(pu)[14])) A.fail(u, TECDSA_ST_PROOF);
    U256 sum = sc_add(u256_load(A.p(F_DELTA, u)), u256_load(A.p(F_DELTA, pu)));
    if (u256_is_zero(sum)) A.fail(u, TECDSA_ST_PROOF);          // reference: .unwrap() panic on a zero sum
    u256_store(A.p(F_DINV, u), sc_inv(sum));
}

// ------------------------------------------------------------------------------ round 4
// SignKeys::phase4 (party_i.rs:642-687), R_dash (sign/rounds.rs:452), first half of PDLwSlackProof::prove
// (utilities/zk_pdl_with_slack/mod.rs:85-92)
static __global__ void gg20_r4_pre(Arena A) {
    int u = blockIdx.x * blockDim.x + threadIdx.x;
    if (u >= A.U) return;
    const int pu = A.peer[u];
    const uint32_t* rnd = A.p(F_RND, u);
    Affine gg_own = affine_load(A.p(F_GG, u)), gg_peer = affine_load(A.p(F_GG, pu));
    uint32_t com[8];
    hash_commit_point(com, gg_peer, A.p(F_RND, pu) + RND_BLIND);
    bool ok = affine_eq(affine_load(A.p(F_DL0, pu)), gg_peer) && st::cmp(com, A.p(F_COM, pu), 8) == 0;
    if (!ok) A.fail(u, TECDSA_ST_COMMITMENT);
    // R is bit-identical on the two units of a session, which lets one unit's PDL and HomoElGamal verdicts stand for both: the
    // operand order of the sum and the per-unit k and alpha change only the projective representation and the other two
    // outputs of the shared inversion, and the affine R is the unique (X/Z^2, Y/Z^3) or the identity (tests/test_session_verdicts.py)
    const Jac Rj = jac_mul(j_add_aff(gg_own, gg_peer), u256_load(A.p(F_DINV, u)));
    // R_dash and u1 are multiples of R: they are computed from the projective R and all three are normalised together
    Affine R, Rd, U1;
    jac_to_affine3(R, Rd, U1, Rj, jac_mul(Rj, load_scalar(rnd + RND_K)), jac_mul(Rj, sc_from_limbs(rnd + RND_PDL_ALPHA, 24)));
    affine_store(A.p(F_R, u), R);
    affine_store(A.p(F_RD, u), Rd);
    affine_store(A.p(F_PU1, u), U1);
    uint32_t one = 1;
    st::mul_add(A.p(F_PLIN, u), 128, rnd + RND_PDL_ALPHA, 24, A.k(KT_N, A.row_own[u]), 64, &one, 1);
}

static __global__ void gg20_r4_mid(Arena A) {
    int u = blockIdx.x * blockDim.x + threadIdx.x;
    if (u >= A.U) return;
    const uint32_t* rnd = A.p(F_RND, u);
    uint32_t* e = A.p(F_PE, u);
    pdl_hash(e, affine_load(A.p(F_R, u)), affine_load(A.p(F_RD, u)), A.p(F_CK, u), A.p(F_PZ, u), affine_load(A.p(F_PU1, u)),
             A.p(F_PU2, u), A.p(F_PU3, u));
    st::mul_add(A.p(F_PS1, u), 28, e, 8, rnd + RND_K, 8, rnd + RND_PDL_ALPHA, 24);          // s1 = e*x + alpha (:112)
    st::mul_add(A.p(F_PS3, u), 92, e, 8, rnd + RND_PDL_RHO, 72, rnd + RND_PDL_GAMMA, 88);   // s3 = e*rho + gamma (:114)
}

// ------------------------------------------------------------------------------ round 5
// PDLwSlackProof::verify of the unit's own proof (party_i.rs:719-766 -> zk_pdl_with_slack/mod.rs:127-179), the check the
// reference runs on the prover's side (sign/rounds.rs:546-558).  Its one verifier-side input, R, is bit-identical on the two
// units of a session (gg20_r4_pre), so the verdict is the peer's verdict on this proof too.
static __global__ void gg20_r5_pre(Arena A) {
    int u = blockIdx.x * blockDim.x + threadIdx.x;
    if (u >= A.U) return;
    uint32_t one = 1;
    pdl_hash(A.p(F_VE0, u), affine_load(A.p(F_R, u)), affine_load(A.p(F_RD, u)), A.p(F_CK, u), A.p(F_PZ, u), affine_load(A.p(F_PU1, u)),
             A.p(F_PU2, u), A.p(F_PU3, u));
    st::mul_add(A.p(F_VLIN0, u), 128, A.p(F_PS1, u), 28, A.k(KT_N, A.row_own[u]), 64, &one, 1);
}

// the EC relation and the two big-integer comparisons of PDLwSlackProof::verify
static __global__ void gg20_r5_check(Arena A) {
    int u = blockIdx.x * blockDim.x + threadIdx.x;
    if (u >= A.U) return;
    const uint8_t* fl = A.flags(u);
    Affine R = affine_load(A.p(F_R, u));
    U256 e = sc_from_limbs(A.p(F_VE0, u), 8);
    U256 s1 = sc_from_limbs(A.p(F_PS1, u), 28);
    const Jac u1t = j_lin2(R, s1, affine_load(A.p(F_RD, u)), sc_neg(e));
    bool ok = fl[6] && fl[8];                         // z^e mod N_tilde and the prover's ciphertext mod N^2 invertible
    ok = ok && jac_eq_affine(u1t, affine_load(A.p(F_PU1, u)));
    ok = ok && st::cmp(A.p(F_VU20, u), A.p(F_PU2, u), 128) == 0;
    ok = ok && st::cmp(A.p(F_VU30, u), A.p(F_PU3, u), 64) == 0;
    A.flags(u)[16] = ok;
}

static __global__ void gg20_r5_finish(Arena A) {
    int u = blockIdx.x * blockDim.x + threadIdx.x;
    if (u >= A.U) return;
    const int pu = A.peer[u];
    const uint32_t* rnd = A.p(F_RND, u);
    Affine R = affine_load(A.p(F_R, u));
    if (!(A.flags(u)[16] && A.flags(pu)[16])) A.fail(u, TECDSA_ST_PDL_VERIFY);
    // phase5_check_R_dash_sum (party_i.rs:768-776): G + sum(R_dash) - G == G
    if (!jac_eq_affine(j_add_aff(affine_load(A.p(F_RD, u)), affine_load(A.p(F_RD, pu))), affine_G())) A.fail(u, TECDSA_ST_PHASE5_BAD_SUM);
    // phase6_compute_S_i_and_proof_of_consistency (party_i.rs:778-799)
    const U256 sigma = u256_load(A.p(F_SIGMA, u)), l = load_scalar(rnd + RND_L);
    const U256 s1 = load_scalar(rnd + RND_HEG_S1), s2 = load_scalar(rnd + RND_HEG_S2);
    Affine S, T, A3;                                 // S_i = R*sigma, A1 + A2 = H*s1 + G*s2, A3 = R*s2: one shared inversion
    {
        const Jac Rj = jac_from_affine(R);
        jac_to_affine3(S, T, A3, jac_mul(Rj, sigma), j_lin_GH(s2, s1), jac_mul(Rj, s2));
    }
    affine_store(A.p(F_SI, u), S);
    U256 e = heg_hash(T, A3, R, affine_load(A.p(F_T, u)), S);
    uint32_t* heg = A.p(F_HEG, u);
    affine_store(heg, T); affine_store(heg + 16, A3);
    u256_store(heg + 32, u256_is_zero(l) ? s1 : sc_add(s1, sc_mul(l, e)));
    u256_store(heg + 40, sc_add(s2, sc_mul(sigma, e)));
}

// phase6_verify_proof + phase6_check_S_i_sum (party_i.rs:801-848), then the unit's result record:
// a SHA-256 over every message it emitted, in the fixed-width encoding of oracle/gg20_oracle.py
// HomoELGamalProof::verify of the unit's own proof (party_i.rs:801-833); R is the session's R, bit-identical on both units
static __global__ void gg20_r6_check(Arena A) {
    int u = blockIdx.x * blockDim.x + threadIdx.x;
    if (u >= A.U) return;
    A.flags(u)[18] = heg_verify(A.p(F_HEG, u), affine_load(A.p(F_R, u)), affine_load(A.p(F_T, u)), affine_load(A.p(F_SI, u)));
}

static __global__ void gg20_r6(Arena A) {
    int u = blockIdx.x * blockDim.x + threadIdx.x;
    if (u >= A.U) return;
    const int pu = A.peer[u];
    if (!(A.flags(u)[18] && A.flags(pu)[18])) A.fail(u, TECDSA_ST_PHASE6);
    if (!jac_eq_affine(j_add_aff(affine_load(A.p(F_SI, u)), affine_load(A.p(F_SI, pu))), affine_load(A.ypk + (size_t)A.keyset[u] * 16))) A.fail(u, TECDSA_ST_PHASE6);

    Sha256 h; h.init();
    const uint32_t* rnd = A.p(F_RND, u);
    // M1: MessageA + commitment
    h.put_fixed(A.p(F_CK, u), 128);
    for (int x = 0; x < 3; x++) {
        h.put_fixed(A.p(F_Z0 + x, u), 64); h.put_fixed(A.p(F_E0 + x, u), 8); h.put_fixed(A.p(F_S0 + x, u), 64);
        put_padded(h, A.p(F_S10 + x, u), 28, 32); put_padded(h, A.p(F_S20 + x, u), 92, 96);
    }
    h.put_fixed(A.p(F_COM, u), 8);
    // M2: the two MessageB
    for (int m = 0; m < 2; m++) {
        h.put_fixed(A.p(m ? F_CBW : F_CBG, u), 128);
        for (int d = 0; d < 2; d++) {
            const uint32_t* dl = A.p(F_DL0 + 2 * m + d, u);
            put_point33(h, dl); put_point33(h, dl + 16); h.put_fixed(dl + 32, 8);
        }
    }
    // M3
    const uint32_t* ped = A.p(F_PED, u);
    h.put_fixed(A.p(F_DELTA, u), 8); put_point33(h, A.p(F_T, u)); h.put_fixed(ped, 8);
    put_point33(h, ped + 8); put_point33(h, ped + 24); put_point33(h, A.p(F_T, u));
    h.put_fixed(ped + 40, 8); h.put_fixed(ped + 48, 8);
    // M4
    h.put_fixed(rnd + RND_BLIND, 8); put_point33(h, A.p(F_GG, u));
    // M5
    put_point33(h, A.p(F_RD, u)); h.put_fixed(A.p(F_PZ, u), 64); put_point33(h, A.p(F_PU1, u));
    h.put_fixed(A.p(F_PU2, u), 128); h.put_fixed(A.p(F_PU3, u), 64);
    put_padded(h, A.p(F_PS1, u), 28, 32); h.put_fixed(A.p(F_PS2, u), 64); put_padded(h, A.p(F_PS3, u), 92, 96);
    // M6
    const uint32_t* heg = A.p(F_HEG, u);
    put_point33(h, A.p(F_SI, u)); put_point33(h, heg); put_point33(h, heg + 16);
    h.put_fixed(heg + 32, 8); h.put_fixed(heg + 40, 8);
    h.finish(A.p(F_DIGEST, u));
}

// ------------------------------------------------------------------------------ per-key constants
// One thread per key row: N^2, p^2, q^2, p-1, q-1 and the CRT constants of Paillier decrypt.
static __global__ void gg20_key_setup(uint32_t* const* tables, int rows) {
    int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= rows) return;
    auto T = [&](int t) { return tables[t] + (size_t)r * KEY_SIZE_D[t]; };
    const uint32_t *p = T(KT_P), *q = T(KT_Q);
    st::mul(T(KT_N), p, 32, q, 32);
    st::mul(T(KT_NN), T(KT_N), 64, T(KT_N), 64);
    st::mul(T(KT_PP), p, 32, p, 32);
    st::mul(T(KT_QQ), q, 32, q, 32);
    uint32_t one[32]; st::zero(one, 32); one[0] = 1;
    st::sub(T(KT_PM1), p, one, 32);
    st::sub(T(KT_QM1), q, one, 32);
    st::mod_slow(T(KT_QMODPM1), q, 32, T(KT_PM1), 32);
    st::mod_slow(T(KT_PMODQM1), p, 32, T(KT_QM1), 32);
    uint32_t scratch[65], t1[32], t2[32], rr[32], x[32], acc[32];
    for (int half = 0; half < 2; half++) {
        const uint32_t* m = half ? q : p;        // modulus
        const uint32_t* o = half ? p : q;        // the other prime
        // m^-1 mod 2^1024 by Newton/Hensel lifting: x <- x * (2 - m*x)
        uint32_t* inv2 = T(half ? KT_QINV2 : KT_PINV2);
        st::zero(x, 32); x[0] = 0u - st::neg_inv32_st(m[0]);
        for (int it = 0; it < 6; it++) {
            st::mul_low(t1, m, x, 32);
            uint32_t two[32]; st::zero(two, 32); two[0] = 2;
            st::sub(t2, two, t1, 32);
            st::mul_low(t1, x, t2, 32);
            st::copy(x, t1, 32);
        }
        st::copy(inv2, x, 32);
        // Montgomery domain mod m: R^2
        const uint32_t m0 = st::neg_inv32_st(m[0]);
        st::r_mod_m(rr, m, 32);
        for (int i = 0; i < 1024; i++) {
            uint32_t top = rr[31] >> 31;
            for (int j = 31; j > 0; j--) rr[j] = (rr[j] << 1) | (rr[j - 1] >> 31);
            rr[0] <<= 1;
            if (top || st::cmp(rr, m, 32) >= 0) st::sub(rr, rr, m, 32);
        }
        // (o mod m)^-1 in Montgomery form via Fermat: (oR)^(m-2)
        st::mod_slow(t1, o, 32, m, 32);
        st::mont_mul(t1, t1, rr, m, m0, 32, scratch);           // o*R
        uint32_t em2[32], twov[32]; st::zero(twov, 32); twov[0] = 2;
        st::sub(em2, m, twov, 32);
        st::r_mod_m(acc, m, 32);                                // 1*R
        for (int i = 1023; i >= 0; i--) {
            st::mont_mul(acc, acc, acc, m, m0, 32, scratch);
            if ((em2[i >> 5] >> (i & 31)) & 1u) st::mont_mul(acc, acc, t1, m, m0, 32, scratch);
        }
        // acc = (o^-1 mod m) * R mod m
        if (half == 0) {
            // hp = (-q)^-1 mod p  ->  hp*R = p - acc
            st::sub(T(KT_HPR), p, acc, 32);
        } else {
            st::sub(T(KT_HQR), q, acc, 32);      // hq = (-p)^-1 mod q
            st::copy(T(KT_PINVQR), acc, 32);     // (p^-1 mod q) * R
        }
    }
    // ((p^2)^-1 mod q^2) * R64 mod q^2, R64 = 2^2048: lift p^-1 mod q to mod q^2 (Newton), square.
    {
        const uint32_t* qq = T(KT_QQ);
        const uint32_t m0 = st::neg_inv32_st(qq[0]);
        uint32_t rr64[64], big[129], pM[64], xM[64], tM[64], two[64], ext[64];
        st::r_mod_m(rr64, qq, 64);
        st::copy(two, rr64, 64);                                  // 1*R
        {   // two = 2*R mod q^2
            uint32_t top = two[63] >> 31;
            for (int j = 63; j > 0; j--) two[j] = (two[j] << 1) | (two[j - 1] >> 31);
            two[0] <<= 1;
            if (top || st::cmp(two, qq, 64) >= 0) st::sub(two, two, qq, 64);
        }
        for (int i = 0; i < 2048; i++) {                          // rr64 = R^2 mod q^2
            uint32_t top = rr64[63] >> 31;
            for (int j = 63; j > 0; j--) rr64[j] = (rr64[j] << 1) | (rr64[j - 1] >> 31);
            rr64[0] <<= 1;
            if (top || st::cmp(rr64, qq, 64) >= 0) st::sub(rr64, rr64, qq, 64);
        }
        st::zero(ext, 64); st::copy(ext, p, 32);
        st::mont_mul(pM, ext, rr64, qq, m0, 64, big);             // p * R
        // x0 = p^-1 mod q (plain) from its Montgomery form mod q
        uint32_t x0[32], one32[32], sc[65];
        st::zero(one32, 32); one32[0] = 1;
        st::mont_mul(x0, T(KT_PINVQR), one32, q, st::neg_inv32_st(q[0]), 32, sc);
        st::zero(ext, 64); st::copy(ext, x0, 32);
        st::mont_mul(xM, ext, rr64, qq, m0, 64, big);             // x0 * R
        st::mont_mul(tM, pM, xM, qq, m0, 64, big);                // p*x0 * R
        if (st::sub(tM, two, tM, 64)) st::add(tM, tM, qq, 64);    // (2 - p*x0) * R mod q^2
        st::mont_mul(xM, xM, tM, qq, m0, 64, big);                // x1 * R,  x1 = p^-1 mod q^2
        st::mont_mul(T(KT_PPINVQQR), xM, xM, qq, m0, 64, big);    // x1^2 * R = (p^2)^-1 * R mod q^2
    }
}

// recombine `count` (1..4) consecutive (YP, YQ) field pairs starting at slot `first` under the key row rows[u] (the unit's own
// or its peer's) into the consecutive fields starting at `dst`
static __global__ void gg20_crt(Arena A, const uint32_t* rows, int first, int count, int dst) {
    int u = blockIdx.x * blockDim.x + threadIdx.x;
    if (u >= A.U) return;
    const uint32_t row = rows[u];
    for (int s = 0; s < count; s++) crt_combine(A.p(dst + s, u), A, row, A.p(F_YP0 + first + s, u), A.p(F_YQ0 + first + s, u));
}

}  // namespace tecdsa
