// Per-element kernels of the GG18 phase 4 / 5a-5d entry points (gg18.cu): secp256k1 and SHA-256 only, one thread per element.
// Device code only (no runtime calls), so that tests/host_harness can compile it for the CPU.
#pragma once
#include "gg20_glue.cuh"

namespace tecdsa {
namespace gg18 {

__device__ __forceinline__ bool good_point(const Affine& P) { return !P.inf && on_curve(P); }
__device__ __forceinline__ bool u256_gt(const U256& a, const U256& b) {
    for (int i = 7; i >= 0; i--) { if (a.v[i] != b.v[i]) return a.v[i] > b.v[i]; }
    return false;
}
__device__ __forceinline__ bool limbs_eq8(const uint32_t* a, const uint32_t* b) {
    uint32_t x = 0;
    for (int j = 0; j < 8; j++) x |= a[j] ^ b[j];
    return x == 0;
}
// curv HomoELGamalProof [R] for a general statement (G, H, Y = generator, D, E): e = H(T, A3, G, H, Y, D, E)
__device__ __noinline__ U256 heg_hash_general(const Affine& T, const Affine& A3, const Affine& Gp, const Affine& Hp, const Affine& D, const Affine& E) {
    Affine pts[7];
    pts[0] = T; pts[1] = A3; pts[2] = Gp; pts[3] = Hp; pts[4] = affine_G(); pts[5] = D; pts[6] = E;
    return hash_points_scalar(pts, 7);
}
__device__ __forceinline__ Affine neg_affine(const Affine& a) { Affine r = a; if (!a.inf) r.y = fe_neg(a.y); return r; }

// ---- phase 4 (party_i.rs:455-485): for every signer j of the session, b_proof[j].pk == g_gamma_j and the phase-1 commitment of j
// reopens; then R = delta_inv * sum_j g_gamma_j.  b_pk is per element an array of `parties` DLogProof public keys (entry j = the
// pk of the MessageB proof the element received from signer j; for j = itself its own g^gamma, as gg_2018/test.rs passes it).
__global__ void k_gg18_phase4(int parties, const uint32_t* delta_inv, const uint32_t* b_pk16, const uint32_t* g_gamma16, const uint32_t* blind8,
                              const uint32_t* com8, uint32_t* R16, uint8_t* status, int count) {
    int u = blockIdx.x * blockDim.x + threadIdx.x;
    if (u >= count) return;
    const int s0 = (u / parties) * parties;
    bool ok = true;
    Jac acc = jac_identity();
    for (int j = 0; j < parties; j++) {
        const int v = s0 + j;
        const Affine gg = affine_load(g_gamma16 + (size_t)v * 16);
        if (!good_point(gg)) { ok = false; continue; }
        acc = jac_madd(acc, gg);
        const Affine pk = affine_load(b_pk16 + ((size_t)u * parties + j) * 16);
        uint32_t t[8];
        hash_commit_point(t, gg, blind8 + (size_t)v * 8);
        ok = ok && !pk.inf && u256_eq(pk.x, gg.x) && u256_eq(pk.y, gg.y) && limbs_eq8(t, com8 + (size_t)v * 8);
    }
    Affine R = affine_inf();
    const U256 di = load_scalar(delta_inv + (size_t)u * 8);
    if (ok && !jac_is_inf(acc) && !u256_is_zero(di)) R = jac_to_affine(jac_mul(acc, di));
    if (R.inf) ok = false;
    affine_store(R16 + (size_t)u * 16, R);
    status[u] = ok ? TECDSA_ST_OK : TECDSA_ST_INVALID_KEY;
}

// ---- phase 5a/5b (party_i.rs:513-558): A = rho G, B = (l rho) G, V = s R + l G, com = commit(H(V, A, B); blind),
// HomoELGamalProof for (G = A, H = R, Y = g, D = V, E = B) with witness (x = s_i, r = l_i), DLogProof of rho
__global__ void k_gg18_phase5a(const uint32_t* R16, const uint32_t* s8, const uint32_t* l8, const uint32_t* rho8, const uint32_t* blind8,
                               const uint32_t* hs1, const uint32_t* hs2, const uint32_t* dnonce, uint32_t* com8, uint32_t* vab48, uint32_t* heg48,
                               uint32_t* dlog40, uint8_t* status, int count) {
    int u = blockIdx.x * blockDim.x + threadIdx.x;
    if (u >= count) return;
    const Affine R = affine_load(R16 + (size_t)u * 16);
    const U256 s = load_scalar(s8 + (size_t)u * 8), l = load_scalar(l8 + (size_t)u * 8), rho = load_scalar(rho8 + (size_t)u * 8);
    const U256 s1 = load_scalar(hs1 + (size_t)u * 8), s2 = load_scalar(hs2 + (size_t)u * 8);
    if (!good_point(R) || u256_is_zero(rho) || u256_is_zero(l) || u256_is_zero(s2) || u256_is_zero(load_scalar(dnonce + (size_t)u * 8))) {
        status[u] = TECDSA_ST_INVALID_KEY;                        // identity points have no place in the messages (Scalar::random() != 0)
        return;
    }
    Affine pts[3];                                                // V, A, B
    const Jac RJ = jac_from_affine(R);
    const Jac Vj = jac_add(jac_mul(RJ, s), jac_mul_fixed(0, l));
    if (jac_is_inf(Vj)) { status[u] = TECDSA_ST_INVALID_KEY; return; }
    jac_to_affine3(pts[0], pts[1], pts[2], Vj, jac_mul_fixed(0, rho), jac_mul_fixed(0, sc_mul(l, rho)));
    commit_points(com8 + (size_t)u * 8, pts, 3, blind8 + (size_t)u * 8);
    uint32_t* o = vab48 + (size_t)u * 48;
    affine_store(o, pts[0]); affine_store(o + 16, pts[1]); affine_store(o + 32, pts[2]);
    // HomoELGamalProof::prove [R]: A1 = H s1, A2 = Y s2, A3 = G s2, T = A1 + A2, z1 = s1 + x e, z2 = s2 + r e
    const Jac Tj = jac_add(jac_mul(RJ, s1), jac_mul_fixed(0, s2));
    Affine T, A3;
    if (jac_is_inf(Tj)) { status[u] = TECDSA_ST_INVALID_KEY; return; }
    jac_to_affine2(T, A3, Tj, jac_mul(jac_from_affine(pts[1]), s2));
    const U256 e = heg_hash_general(T, A3, pts[1], R, pts[0], pts[2]);
    uint32_t* h = heg48 + (size_t)u * 48;
    affine_store(h, T); affine_store(h + 16, A3);
    u256_store(h + 32, u256_is_zero(s) ? s1 : sc_add(s1, sc_mul(s, e)));
    u256_store(h + 40, sc_add(s2, sc_mul(l, e)));
    dlog_prove(dlog40 + (size_t)u * 40, rho, load_scalar(dnonce + (size_t)u * 8));
    status[u] = TECDSA_ST_OK;
}

// HomoELGamalProof::verify [R]: H z1 + Y z2 == T + D e  and  G z2 == A3 + E e
__device__ __noinline__ bool heg_verify_general(const uint32_t* heg, const Affine& Gp, const Affine& Hp, const Affine& D, const Affine& E) {
    const Affine T = affine_load(heg), A3 = affine_load(heg + 16);
    if (!good_point(T) || !good_point(A3) || !good_point(Gp) || !good_point(Hp) || !good_point(D) || !good_point(E)) return false;
    const U256 z1 = load_scalar(heg + 32), z2 = load_scalar(heg + 40);
    const U256 e = heg_hash_general(T, A3, Gp, Hp, D, E);
    const bool ok1 = jac_eq(jac_add(jac_mul(jac_from_affine(Hp), z1), jac_mul_fixed(0, z2)), jac_madd(jac_mul(jac_from_affine(D), e), T));
    const bool ok2 = jac_eq(jac_mul(jac_from_affine(Gp), z2), jac_madd(jac_mul(jac_from_affine(E), e), A3));
    return ok1 && ok2;
}

// ---- phase 5c's checks of one sender's 5a message, run once per sender (party_i.rs:580-600): its commitment reopens to
// (V, A, B), its HomoELGamalProof holds for (G = A, H = R, Y = g, D = V, E = B) and its DLogProof of rho holds.  verdict[v] = 1
// when all three hold.  Each check is deterministic in the sender's message and R; R is the same on every member of a session that
// passed phase 4 (k_gg18_phase4 derives it from session-wide values), so the sender's own R stands for every receiver's.
__global__ void k_gg18_phase5c_senders(const uint32_t* R16, const uint32_t* com8, const uint32_t* vab48, const uint32_t* blind1, const uint32_t* heg48,
                                       const uint32_t* dlog40, uint8_t* verdict, int count) {
    int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= count) return;
    const uint32_t* d = vab48 + (size_t)v * 48;
    Affine pts[3];
    pts[0] = affine_load(d); pts[1] = affine_load(d + 16); pts[2] = affine_load(d + 32);
    bool ok = good_point(pts[0]) && good_point(pts[1]) && good_point(pts[2]);
    if (ok) {
        uint32_t t[8];
        commit_points(t, pts, 3, blind1 + (size_t)v * 8);
        ok = limbs_eq8(t, com8 + (size_t)v * 8) && heg_verify_general(heg48 + (size_t)v * 48, pts[1], affine_load(R16 + (size_t)v * 16), pts[0], pts[2]) &&
             dlog_verify(dlog40 + (size_t)v * 40);
    }
    verdict[v] = ok ? 1 : 0;
}

// ---- phase 5c (party_i.rs:560-629) ------------------------------------------------------------------------------------
// sender_ok = NULL: every element checks every other signer's 5a message itself.  Otherwise sender_ok[v] is the verdict of
// k_gg18_phase5c_senders for element v, read in place of the three checks (same com2, decom2 and status when R is the same on
// every member of the session).
__global__ void k_gg18_phase5c(int parties, const uint32_t* R16, const uint32_t* y16, const uint32_t* msg8, const uint32_t* rho8, const uint32_t* l8,
                               const uint32_t* blind2, const uint32_t* com8, const uint32_t* vab48, const uint32_t* blind1, const uint32_t* heg48,
                               const uint32_t* dlog40, uint32_t* com2, uint32_t* ut32, uint8_t* status, int count, const uint8_t* sender_ok = nullptr) {
    int u = blockIdx.x * blockDim.x + threadIdx.x;
    if (u >= count) return;
    const int s0 = (u / parties) * parties;
    const Affine R = affine_load(R16 + (size_t)u * 16), Y = affine_load(y16 + (size_t)u * 16);
    bool ok = true, rep = good_point(R) && good_point(Y);
    Jac vsum = jac_identity(), asum = jac_identity();
    for (int j = 0; j < parties && rep; j++) {
        const int v = s0 + j;
        const uint32_t* d = vab48 + (size_t)v * 48;
        Affine pts[3];
        pts[0] = affine_load(d); pts[1] = affine_load(d + 16); pts[2] = affine_load(d + 32);
        if (!good_point(pts[0]) || !good_point(pts[1]) || !good_point(pts[2])) { if (v == u) rep = false; else ok = false; continue; }
        vsum = jac_madd(vsum, pts[0]);
        if (v == u) continue;                                     // own V_i joins the sum; only the others' messages are checked
        asum = jac_madd(asum, pts[1]);
        if (sender_ok) {
            if (!sender_ok[v]) ok = false;
            continue;
        }
        uint32_t t[8];
        commit_points(t, pts, 3, blind1 + (size_t)v * 8);
        if (!limbs_eq8(t, com8 + (size_t)v * 8)) ok = false;
        else if (!heg_verify_general(heg48 + (size_t)v * 48, pts[1], R, pts[0], pts[2])) ok = false;
        else if (!dlog_verify(dlog40 + (size_t)v * 40)) ok = false;
    }
    uint8_t st = TECDSA_ST_OK;
    uint32_t* o = ut32 + (size_t)u * 32;
    for (int j = 0; j < 32; j++) o[j] = 0;
    for (int j = 0; j < 8; j++) com2[(size_t)u * 8 + j] = 0;
    if (!rep) st = TECDSA_ST_INVALID_SIG;
    else {
        // v = v_i + sum V_j - m G - r y;  u_i = rho v;  t_i = l a
        const U256 r = sc_reduce_once(R.x, 0), m = sc_from_limbs(msg8 + (size_t)u * 8, 8);
        Jac vj = jac_add(vsum, jac_mul_fixed(0, sc_neg(m)));
        vj = jac_add(vj, jac_mul(jac_from_affine(neg_affine(Y)), r));
        const Jac uj = jac_mul(vj, load_scalar(rho8 + (size_t)u * 8)), tj = jac_mul(asum, load_scalar(l8 + (size_t)u * 8));
        if (jac_is_inf(uj) || jac_is_inf(tj)) st = TECDSA_ST_INVALID_SIG;          // identity: no recallable encoding in the hash
        else {
            Affine pts[2];
            jac_to_affine2(pts[0], pts[1], uj, tj);
            if (!ok) st = TECDSA_ST_COMMITMENT;                                     // Err(InvalidCom)
            else {
                commit_points(com2 + (size_t)u * 8, pts, 2, blind2 + (size_t)u * 8);
                affine_store(o, pts[0]); affine_store(o + 16, pts[1]);
            }
        }
    }
    status[u] = st;
}

// ---- phase 5d (party_i.rs:631-665): every second commitment reopens, and g + sum t + sum B - sum u == g --------------------
__global__ void k_gg18_phase5d(int parties, const uint32_t* ut32, const uint32_t* blind2, const uint32_t* com2, const uint32_t* vab48, uint8_t* status, int count) {
    int u = blockIdx.x * blockDim.x + threadIdx.x;
    if (u >= count) return;
    const int s0 = (u / parties) * parties;
    bool com_ok = true, pts_ok = true;
    Jac plus = jac_from_affine(affine_G()), minus = jac_identity();
    for (int j = 0; j < parties; j++) {
        const int v = s0 + j;
        Affine pts[2];
        pts[0] = affine_load(ut32 + (size_t)v * 32); pts[1] = affine_load(ut32 + (size_t)v * 32 + 16);
        const Affine B = affine_load(vab48 + (size_t)v * 48 + 32);
        if (!good_point(pts[0]) || !good_point(pts[1]) || !good_point(B)) { pts_ok = false; continue; }
        uint32_t t[8];
        commit_points(t, pts, 2, blind2 + (size_t)v * 8);
        com_ok = com_ok && limbs_eq8(t, com2 + (size_t)v * 8);
        plus = jac_madd(jac_madd(plus, pts[1]), B);
        minus = jac_madd(minus, pts[0]);
    }
    uint8_t st = TECDSA_ST_OK;
    if (!pts_ok || !com_ok) st = TECDSA_ST_COMMITMENT;                              // Err(InvalidCom)
    else {
        // plus - minus == g  <=>  plus == g + minus
        if (!jac_eq(plus, jac_madd(minus, affine_G()))) st = TECDSA_ST_INVALID_KEY;  // Err(InvalidKey)
    }
    status[u] = st;
}

// ---- phase5_local_sig (:489-511): s_i = m k_i + r sigma_i -------------------------------------------------------------------
__global__ void k_gg18_local_sig(const uint32_t* msg8, const uint32_t* R16, const uint32_t* k8, const uint32_t* sigma8, uint32_t* s8, int count) {
    int u = blockIdx.x * blockDim.x + threadIdx.x;
    if (u >= count) return;
    const U256 r = sc_reduce_once(u256_load(R16 + (size_t)u * 16), 0);
    u256_store(s8 + (size_t)u * 8, sc_add(sc_mul(sc_from_limbs(msg8 + (size_t)u * 8, 8), load_scalar(k8 + (size_t)u * 8)), sc_mul(r, load_scalar(sigma8 + (size_t)u * 8))));
}

// ---- output_signature (:666-703) + verify (:706-730), one thread per element (every signer derives the same signature) -------
__global__ void k_gg18_output(int parties, const uint32_t* R16, const uint32_t* y16, const uint32_t* msg8, const uint32_t* s8, uint32_t* sig_r,
                              uint32_t* sig_s, uint8_t* recid, uint8_t* status, int count) {
    int u = blockIdx.x * blockDim.x + threadIdx.x;
    if (u >= count) return;
    const int s0 = (u / parties) * parties;
    U256 sum = u256_zero();
    for (int j = 0; j < parties; j++) sum = sc_add(sum, load_scalar(s8 + (size_t)(s0 + j) * 8));
    const Affine R = affine_load(R16 + (size_t)u * 16), Y = affine_load(y16 + (size_t)u * 16);
    const U256 r = sc_reduce_once(R.x, 0);
    uint8_t rid = (uint8_t)(sc_reduce_once(R.y, 0).v[0] & 1u);
    const U256 neg = sc_neg(sum);
    if (u256_gt(sum, neg)) { sum = neg; rid ^= 1; }
    u256_store(sig_r + (size_t)u * 8, r); u256_store(sig_s + (size_t)u * 8, sum);
    recid[u] = rid;
    bool ok = good_point(R) && good_point(Y) && !u256_is_zero(sum);
    if (ok) {
        const U256 b = sc_inv(sum);
        const Affine P = lin_GP(sc_mul(sc_from_limbs(msg8 + (size_t)u * 8, 8), b), Y, sc_mul(r, b));
        ok = !P.inf && u256_eq(sc_reduce_once(P.x, 0), r);
    }
    status[u] = ok ? TECDSA_ST_OK : TECDSA_ST_INVALID_SIG;
}


}  // namespace gg18
}  // namespace tecdsa
