// TEST INFRASTRUCTURE: compiles the per-element, per-pair and per-session kernels of the GG20 offline stage for any signing set
// (csrc/gg20_general_kernels.cuh) for the HOST with shims for the CUDA qualifiers (the technique of harness.cpp), so that the CPU
// test-suite can check them against the oracle without a GPU.  Each h_* function runs one kernel over every thread of its launch.
// Nothing here is reachable from the product library.
#include <cstdint>
#include <cstdio>
#include <cstring>
#define __device__
#define __forceinline__ inline
#define __noinline__
#define __constant__
#define __global__
static inline uint32_t __funnelshift_r(uint32_t lo, uint32_t hi, int n) { n &= 31; return n ? (lo >> n) | (hi << (32 - n)) : lo; }
static inline int __clz(uint32_t x) { return x ? __builtin_clz(x) : 32; }
struct Dim3 { unsigned x, y, z; };
static Dim3 blockIdx = {0, 0, 0}, blockDim = {1, 1, 1}, threadIdx = {0, 0, 0};
#include "gg20_general_kernels.cuh"
using namespace tecdsa;

template <class F> static void each_thread(int count, F f) {
    blockIdx.x = 0; blockDim.x = (unsigned)count;
    for (int t = 0; t < count; t++) { threadIdx.x = (unsigned)t; f(); }
    threadIdx.x = 0; blockDim.x = 1;
}

static uint32_t g_host_fb[2 * secp::FBP_WINDOWS * secp::FBP_DIGITS * 16];
extern "C" {
void h_init() {
    blockDim.x = 2 * secp::FBP_WINDOWS; blockIdx.x = 0;
    for (int t = 0; t < 2 * secp::FBP_WINDOWS; t++) { threadIdx.x = t; secp::fb_points_build(g_host_fb); }
    secp::g_fb_points = g_host_fb;
    threadIdx.x = 0; blockDim.x = 1;
}
void h_index(const uint32_t* sess, int T, int P, int E, uint32_t* row, uint32_t* st_row, uint32_t* st_elem, uint32_t* pr_me, uint32_t* pr_peer,
             uint32_t* pr_row_peer) {
    const int threads = (P > 2 * (T - 1) ? P : 2 * (T - 1)) * E;
    each_thread(threads, [&] { gen::k_gen_index(sess, T, P, E, row, st_row, st_elem, pr_me, pr_peer, pr_row_peer, threads); });
}
void h_lagrange(const uint32_t* sess, int T, int P, const uint32_t* xi, const uint32_t* pk, uint32_t* w, uint32_t* gw, int count) {
    each_thread(count, [&] { gen::k_gen_lagrange(sess, T, P, xi, pk, w, gw, count); });
}
void h_msgb_status(const uint8_t* pst, int P, int T, int E, uint8_t* pair_st, int np) {
    each_thread(np, [&] { gen::k_gen_msgb_status(pst, P, T, E, pair_st, np); });
}
void h_round1(int T, int E, const uint8_t* st_b, uint8_t* cand) { each_thread(E, [&] { gen::k_gen_round1(T, E, st_b, cand, E); }); }
void h_round2(int T, int E, const uint8_t* st_a, const uint32_t* alpha, const uint32_t* beta, const uint32_t* bp, const uint32_t* gw, const uint32_t* k,
              const uint32_t* gamma, const uint32_t* w, uint32_t* delta, uint32_t* sigma, uint8_t* cand) {
    each_thread(E, [&] { gen::k_gen_round2(T, E, st_a, alpha, beta, bp, gw, k, gamma, w, delta, sigma, cand, E); });
}
void h_round3(int T, const uint32_t* delta, const uint8_t* ped_st, uint32_t* dinv, uint8_t* cand, int sessions) {
    each_thread(sessions, [&] { gen::k_gen_round3(T, delta, ped_st, dinv, cand, sessions); });
}
void h_round5(int T, int E, const uint8_t* pdl_st, const uint32_t* Rd, uint8_t* cand, int sessions) {
    each_thread(sessions, [&] { gen::k_gen_round5(T, E, pdl_st, Rd, cand, sessions); });
}
void h_round6(int T, const uint32_t* sess, const uint8_t* heg_st, const uint32_t* S, const uint32_t* y, uint8_t* cand, int sessions) {
    each_thread(sessions, [&] { gen::k_gen_round6(T, sess, heg_st, S, y, cand, sessions); });
}
void h_round_end(int T, const uint8_t* cand, uint8_t* status, uint8_t* stopped, int sessions) {
    each_thread(sessions, [&] { gen::k_gen_round_end(T, cand, status, stopped, sessions); });
}
void h_finish(int T, const uint8_t* status, const uint8_t* stopped, const uint32_t* R, const uint32_t* sigma, const uint32_t* Tp, uint8_t* st_out,
              uint32_t* R_out, uint32_t* sigma_out, uint32_t* T_out, uint8_t* complete, int count) {
    each_thread(count, [&] { gen::k_gen_finish(T, status, stopped, R, sigma, Tp, st_out, R_out, sigma_out, T_out, complete, count); });
}
}
