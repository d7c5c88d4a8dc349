// TEST INFRASTRUCTURE: compiles the product's seeded sampler (csrc/chacha20.cuh, csrc/sampler.cuh) for the HOST with shims for
// the CUDA qualifiers (the technique of harness.cpp), so that the CPU test-suite can check it against oracle/seeded_sampling.py
// without a GPU.  Nothing here is reachable from the product library.
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
#include "sampler.cuh"
using namespace tecdsa;

extern "C" {
void h_chacha_block(uint32_t* out16, const uint32_t* key8, uint32_t counter, uint32_t n0, uint32_t n1, uint32_t n2) {
    chacha::block_to(out16, 16, key8, counter, n0, n1, n2);
}
// one value; returns 1 / 0 (smp::sample), *attempts = candidates drawn
int h_sample(const uint32_t* key8, uint32_t stream, uint64_t id, int kind, uint32_t* out, int limbs, const uint32_t* bound, int nb, int bits,
             uint32_t cap, uint32_t* attempts) {
    smp::Stream s = smp::open(key8, stream, id);
    const bool ok = smp::sample(s, kind, out, limbs, bound, nb, bits, cap);
    *attempts = s.attempts;
    return ok ? 1 : 0;
}
void h_gg20_sample_bounds(const uint32_t* nt_tab, uint32_t* qnt, uint32_t* q3nt, int rows) {
    for (int r = 0; r < rows; r++) { smp::gg20_sample_bounds(nt_tab, qnt, q3nt, r, 0); smp::gg20_sample_bounds(nt_tab, qnt, q3nt, r, 1); }
}
int h_gg20_sample_field(const uint32_t* key8, uint64_t unit_id, int f, uint32_t own, uint32_t peer, uint32_t row0, const uint32_t* n_tab,
                        const uint32_t* qnt, const uint32_t* q3nt, uint32_t* rec, uint32_t cap) {
    return smp::gg20_sample_field(key8, unit_id, f, own, peer, row0, n_tab, qnt, q3nt, rec, cap) ? 1 : 0;
}
// the whole record of one unit, as k_gg20_sample fills it; returns the number of fields that failed
int h_gg20_sample_unit(const uint32_t* key8, uint64_t unit_id, uint32_t own, uint32_t peer, uint32_t row0, const uint32_t* n_tab, const uint32_t* qnt,
                       const uint32_t* q3nt, uint32_t* rec, uint32_t cap) {
    int bad = 0;
    for (int f = 0; f < TECDSA_RNDS_COUNT; f++) bad += smp::gg20_sample_field(key8, unit_id, f, own, peer, row0, n_tab, qnt, q3nt, rec, cap) ? 0 : 1;
    return bad;
}
}
