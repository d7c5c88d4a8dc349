// TEST INFRASTRUCTURE: compiles the per-unit round kernels of the fused GG20 offline stage (csrc/gg20_rounds.cuh) for the HOST
// with shims for the CUDA qualifiers (the technique of harness.cpp), and runs them over a hand-built arena, so that the CPU
// test-suite can check how a session's two units share proof verdicts and R without a GPU.  The arena is laid out exactly as
// csrc/gg20.cu lays it out (fields in declaration order, each an operand-major array over the units).
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
#include "gg20_rounds.cuh"
using namespace tecdsa;

static uint32_t g_host_fb[2 * secp::FBP_WINDOWS * secp::FBP_DIGITS * 16];

extern "C" {
void h_init() {
    blockDim.x = 2 * secp::FBP_WINDOWS; blockIdx.x = 0;
    for (int t = 0; t < 2 * secp::FBP_WINDOWS; t++) { threadIdx.x = t; secp::fb_points_build(g_host_fb); }
    secp::g_fb_points = g_host_fb;
    threadIdx.x = 0; blockDim.x = 1;
}
int h_field_count() { return F_COUNT; }
const char* h_field_name(int f) { return FIELD_NAME[f]; }
int h_field_size(int f) { return FIELD_SIZE[f]; }

// kernel ids: 0 gg20_r3_check, 1 gg20_r3_finish, 2 gg20_r4_pre, 3 gg20_r5_check, 4 gg20_r5_finish, 5 gg20_r6_check, 6 gg20_r6
// `keys` holds KT_COUNT table pointers (rows as in csrc/gg20.cu), `ypk` 16 limbs per key set
int h_run(int kernel, uint32_t* base, int U, const uint32_t* const* keys, const uint32_t* ypk, const uint32_t* row_own,
          const uint32_t* row_peer, const uint32_t* peer, const uint32_t* keyset, uint8_t* status) {
    Arena A;
    memset(&A, 0, sizeof(A));
    uint32_t limbs = 0;
    for (int f = 0; f < F_COUNT; f++) { A.off[f] = limbs; A.size[f] = (uint16_t)FIELD_SIZE[f]; limbs += FIELD_SIZE[f]; }
    A.base = base; A.U = U;
    for (int t = 0; t < KT_COUNT; t++) A.key[t] = keys[t];
    A.ypk = ypk; A.row_own = row_own; A.row_peer = row_peer; A.peer = peer; A.keyset = keyset; A.status = status;
    void (*const kern[])(Arena) = {gg20_r3_check, gg20_r3_finish, gg20_r4_pre, gg20_r5_check, gg20_r5_finish, gg20_r6_check, gg20_r6};
    if (kernel < 0 || kernel >= (int)(sizeof(kern) / sizeof(kern[0]))) return -1;
    blockIdx.x = 0; blockDim.x = (unsigned)U;
    for (int t = 0; t < U; t++) { threadIdx.x = (unsigned)t; kern[kernel](A); }
    threadIdx.x = 0; blockDim.x = 1;
    return 0;
}
}
