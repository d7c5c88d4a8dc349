// ChaCha20 block function (RFC 8439 section 2.3: 20 rounds, 32-bit block counter in word 12) for sm_90a, one thread per
// keystream.  The generator behind csrc/sampler.cuh: the reference draws from the OS RNG inside `BigInt::sample_below` /
// `Scalar::random`; the engine derives the same distributions from a caller-supplied 32-byte seed.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace tecdsa {
namespace chacha {

__device__ __forceinline__ uint32_t rotl(uint32_t x, int n) { return __funnelshift_r(x, x, 32 - n); }

#define TECDSA_CHACHA_QR(a, b, c, d)                                                      \
    a += b; d ^= a; d = rotl(d, 16); c += d; b ^= c; b = rotl(b, 12);                     \
    a += b; d ^= a; d = rotl(d, 8);  c += d; b ^= c; b = rotl(b, 7)

// The first n (<= 16) little-endian words of the block (key, counter, nonce = n0 | n1 | n2) written straight to out: the
// state stays in registers, so no local block buffer exists that a caller would have to read back.
__device__ __forceinline__ void block_to(uint32_t* out, int n, const uint32_t* key, uint32_t counter, uint32_t n0, uint32_t n1, uint32_t n2) {
    uint32_t s[16] = {0x61707865u, 0x3320646Eu, 0x79622D32u, 0x6B206574u, key[0], key[1], key[2], key[3],
                      key[4], key[5], key[6], key[7], counter, n0, n1, n2};
    uint32_t x[16];
#pragma unroll
    for (int i = 0; i < 16; i++) x[i] = s[i];
#pragma unroll 1
    for (int r = 0; r < 10; r++) {
        TECDSA_CHACHA_QR(x[0], x[4], x[8], x[12]);
        TECDSA_CHACHA_QR(x[1], x[5], x[9], x[13]);
        TECDSA_CHACHA_QR(x[2], x[6], x[10], x[14]);
        TECDSA_CHACHA_QR(x[3], x[7], x[11], x[15]);
        TECDSA_CHACHA_QR(x[0], x[5], x[10], x[15]);
        TECDSA_CHACHA_QR(x[1], x[6], x[11], x[12]);
        TECDSA_CHACHA_QR(x[2], x[7], x[8], x[13]);
        TECDSA_CHACHA_QR(x[3], x[4], x[9], x[14]);
    }
#pragma unroll
    for (int i = 0; i < 16; i++)
        if (i < n) out[i] = x[i] + s[i];
}
#undef TECDSA_CHACHA_QR

}  // namespace chacha
}  // namespace tecdsa
