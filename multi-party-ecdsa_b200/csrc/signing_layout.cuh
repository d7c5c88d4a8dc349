// Element and pair layout of the one-call signing drivers (gg20_general.cu, gg18_signing.cu), shared by their kernel headers.
// Element u = s * T + p is signer position p of session s (T signers); pair j * E + u (E = elements) is "element u towards its
// j-th peer", the peer being position ind(p, j) = j < p ? j : j + 1 of the same session.
// sess = [sessions][1 + T]: the key set, then the keygen index - 1 of every signer position.
// Device code only (no runtime calls), so that tests/host_harness compiles it for the CPU.
#pragma once
#include "gg20_glue.cuh"

namespace tecdsa {
namespace gen {

__device__ __forceinline__ int peer_of(int T, int u, int j) { const int p = u % T; return u - p + (j < p ? j : j + 1); }
// the pair in which element b sends to element v of the same session
__device__ __forceinline__ int pair_to(int T, int E, int b, int v) { const int pb = b % T, pv = v % T; return (pv < pb ? pv : pv - 1) * E + b; }
__device__ __forceinline__ uint32_t key_row(const uint32_t* sess, int T, int P, int u) {
    const uint32_t* d = sess + (size_t)(u / T) * (1 + T);
    return d[0] * (uint32_t)P + d[1 + u % T];
}
__device__ __forceinline__ bool eq16(const uint32_t* a, const uint32_t* b) {
    uint32_t x = 0;
    for (int i = 0; i < 16; i++) x |= a[i] ^ b[i];
    return x == 0;
}

}  // namespace gen
}  // namespace tecdsa
