// TEST INFRASTRUCTURE: compiles the per-element, per-pair and per-group kernels of the GG20 key generation (csrc/keygen_kernels.cuh)
// for the HOST with shims for the CUDA qualifiers (the technique of harness.cpp), so that the CPU test-suite can check them against
// the oracle without a GPU.  Each h_* function runs one kernel over every thread of its launch.  Nothing here is reachable from the
// product library.
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
#include "keygen_kernels.cuh"
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
void h_commit(const uint32_t* comm, int t1, const uint32_t* blind, uint32_t* com, int count) {
    each_thread(count, [&] { kg::k_kg_commit(comm, t1, blind, com, count); });
}
void h_round2(const uint32_t* y, int y_stride, const uint32_t* blind, const uint32_t* com, const uint8_t* st_ck, const uint32_t* n64, const uint32_t* nt64,
              const uint8_t* st_cd, uint8_t* ok2, int count) {
    each_thread(count, [&] { kg::k_kg_round2(y, y_stride, blind, com, st_ck, n64, nt64, st_cd, ok2, count); });
}
void h_validate_pairs(const uint32_t* comm, int t1, const uint32_t* y, int y_stride, const uint32_t* shares, int n, uint8_t* pair_ok, int pairs) {
    each_thread(pairs, [&] { kg::k_kg_validate_pairs(comm, t1, y, y_stride, shares, n, pair_ok, pairs); });
}
void h_xi(const uint32_t* shares, int n, uint32_t* x, int count) { each_thread(count, [&] { kg::k_kg_xi(shares, n, x, count); }); }
void h_dlog_prove(const uint32_t* x, const uint32_t* nonce, uint32_t* proof, int count) {
    each_thread(count, [&] { kg::k_kg_dlog_prove(x, nonce, proof, count); });
}
void h_global_commitments(const uint32_t* comm, int t1, int n, uint32_t* gcomm, int groups) {
    each_thread(groups * t1, [&] { kg::k_kg_global_commitments(comm, t1, n, gcomm, groups); });
}
void h_round4(const uint32_t* gcomm, int t1, int n, const uint32_t* proof, uint8_t* ok4, int count) {
    each_thread(count, [&] { kg::k_kg_round4(gcomm, t1, n, proof, ok4, count); });
}
void h_finish(int n, int t1, const uint8_t* st_nt, const uint8_t* ok2, const uint8_t* pair_ok, const uint8_t* ok4, const uint32_t* proof, const uint32_t* gcomm,
              uint8_t* status, uint64_t* bad, uint8_t* complete, uint32_t* pk, uint32_t* y, uint32_t* x, uint32_t* vss, uint32_t* n64, uint32_t* dlog_st,
              int count) {
    each_thread(count, [&] { kg::k_kg_finish(n, t1, st_nt, ok2, pair_ok, ok4, proof, gcomm, status, bad, complete, pk, y, x, vss, n64, dlog_st, count); });
}
}
