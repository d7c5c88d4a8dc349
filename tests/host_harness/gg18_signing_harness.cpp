// TEST INFRASTRUCTURE: compiles the per-element and per-session kernels of GG18 signing as one call
// (csrc/gg18_signing_kernels.cuh), the GG18 phase-5 kernels it launches (csrc/gg18_kernels.cuh) and the stop rule it shares with the
// GG20 general call (csrc/gg20_general_kernels.cuh) for the HOST with shims for the CUDA qualifiers (the technique of harness.cpp),
// so that the CPU test-suite can check them against the oracle without a GPU.  Each h_* function runs one kernel over every thread
// of its launch.  Nothing here is reachable from the product library.
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
#include "gg18_kernels.cuh"
#include "gg20_general_kernels.cuh"
#include "gg18_signing_kernels.cuh"
using namespace tecdsa;

template <class F> static void each_thread(int count, F f) {
    blockIdx.x = 0; blockDim.x = (unsigned)count;
    for (int t = 0; t < count; t++) { threadIdx.x = (unsigned)t; f(); }
    threadIdx.x = 0; blockDim.x = 1;
}

typedef const uint32_t* CU;
typedef uint32_t* MU;
static uint32_t g_host_fb[2 * secp::FBP_WINDOWS * secp::FBP_DIGITS * 16];
extern "C" {
void h_init() {
    blockDim.x = 2 * secp::FBP_WINDOWS; blockIdx.x = 0;
    for (int t = 0; t < 2 * secp::FBP_WINDOWS; t++) { threadIdx.x = t; secp::fb_points_build(g_host_fb); }
    secp::g_fb_points = g_host_fb;
    threadIdx.x = 0; blockDim.x = 1;
}
void h_session(int T, CU sess, CU message, CU y_tab, MU msg, MU y, int count) {
    each_thread(count, [&] { g18::k_g18_session(T, sess, message, y_tab, msg, y, count); });
}
void h_msgb(int T, int E, const uint8_t* st_b, uint8_t* cand) { each_thread(E, [&] { g18::k_g18_msgb(T, E, st_b, cand, E); }); }
void h_phase2(int T, int E, const uint8_t* st_a, CU alpha, CU beta, CU k, CU gamma, CU w, MU delta, MU sigma, uint8_t* cand) {
    each_thread(E, [&] { g18::k_g18_phase2(T, E, st_a, alpha, beta, k, gamma, w, delta, sigma, cand, E); });
}
void h_phase3(int T, CU delta, MU dinv, uint8_t* cand, int sessions) { each_thread(sessions, [&] { g18::k_g18_phase3(T, delta, dinv, cand, sessions); }); }
void h_round_end(int T, const uint8_t* cand, uint8_t* status, uint8_t* stopped, int sessions) {
    each_thread(sessions, [&] { gen::k_gen_round_end(T, cand, status, stopped, sessions); });
}
void h_finish(int T, const uint8_t* status, const uint8_t* stopped, CU R, CU r, CU s, const uint8_t* rid, uint8_t* st_out, MU R_out, MU sig_r, MU sig_s,
              uint8_t* recid, uint8_t* complete, int count) {
    each_thread(count, [&] { g18::k_g18_finish(T, status, stopped, R, r, s, rid, st_out, R_out, sig_r, sig_s, recid, complete, count); });
}
void h_phase5a(CU R, CU s, CU l, CU rho, CU blind, CU hs1, CU hs2, CU dn, MU com, MU vab, MU heg, MU dlog, uint8_t* st, int count) {
    each_thread(count, [&] { gg18::k_gg18_phase5a(R, s, l, rho, blind, hs1, hs2, dn, com, vab, heg, dlog, st, count); });
}
void h_phase5c_senders(CU R, CU com, CU vab, CU blind1, CU heg, CU dlog, uint8_t* verdict, int count) {
    each_thread(count, [&] { gg18::k_gg18_phase5c_senders(R, com, vab, blind1, heg, dlog, verdict, count); });
}
void h_phase5c(int parties, CU R, CU y, CU msg, CU rho, CU l, CU blind2, CU com, CU vab, CU blind1, CU heg, CU dlog, MU com2, MU ut, uint8_t* st, int count,
               const uint8_t* verdict) {
    each_thread(count, [&] { gg18::k_gg18_phase5c(parties, R, y, msg, rho, l, blind2, com, vab, blind1, heg, dlog, com2, ut, st, count, verdict); });
}
}
