// The reference's sampling calls on a seeded ChaCha20 keystream, one thread per value:
//   BITS(b)    `BigInt::sample(b)`                      gg_2020/party_i.rs:574
//   BELOW(m)   `BigInt::sample_below(m)`                utilities/mta/mod.rs:57,97-98; mta/range_proofs.rs:48-51;
//                                                       zk_pdl_with_slack/mod.rs:73-77
//   UNIT(m)    `SampleFromMultiplicativeGroup`          mta/range_proofs.rs:538-557 (BELOW until gcd(v, m) = 1)
//   RANGE1(m)  `BigInt::sample_range(1, m - 1)`         zk_pdl_with_slack/mod.rs:74 (1 + BELOW(m - 2))
//   SCALAR     `Scalar::<Secp256k1>::random()`          party_i.rs:563,565,628 (BELOW(q) until non-zero)
// (paths relative to /root/reference/src).  Rejection sampling on bit_length(m) bits is exactly uniform and is what the
// reference does; nothing here reduces a wider value modulo m.
//
// Keystream of one value: key = the caller's seed, nonce word 13 = stream id (which field), words 14 | 15 = the 64-bit element
// id, block counter from 0.  One attempt at b bits consumes ceil(b / 512) whole blocks: the first ceil(b / 32) keystream words
// are the little-endian limbs, the top limb is masked to b mod 32 bits, the rest of the last block is discarded.  The generator
// is not the reference's OS RNG, so only the distribution is contractual; this layout (block-aligned attempts, limbs in
// keystream order) is the one with the fewest ways to get wrong for a second implementation.
//
// Candidates are drawn INTO the output row and compared in place.  After `cap` rejected attempts (the kernels pass
// TECDSA_SAMPLE_ATTEMPTS) the value is zeroed and the caller reports TECDSA_ST_SAMPLING: never a spin.
#pragma once
#include "chacha20.cuh"
#include "gg20_glue.cuh"

namespace tecdsa {
namespace smp {

constexpr int MAX_LIMBS = 128;

struct Stream {
    const uint32_t* key;      // 8 words, device memory
    uint32_t stream;          // nonce word 13
    uint32_t id_lo, id_hi;    // nonce words 14, 15
    uint32_t counter;         // next block
    uint32_t attempts;        // candidates drawn so far for this value
};
__device__ __forceinline__ Stream open(const uint32_t* key, uint32_t stream, uint64_t id) {
    return Stream{key, stream, (uint32_t)id, (uint32_t)(id >> 32), 0u, 0u};
}

__device__ __forceinline__ int bit_length(const uint32_t* a, int n) {
    for (int i = n - 1; i >= 0; i--)
        if (a[i]) return 32 * i + 32 - __clz(a[i]);
    return 0;
}
// bit_length(m - 2) for m >= 3: one less than bit_length(m) exactly when m = 2^k or 2^k + 1
__device__ __forceinline__ int bit_length_minus2(const uint32_t* m, int n) {
    const int bl = bit_length(m, n), top = (bl - 1) >> 5;
    uint32_t rest = 0;
    for (int i = 1; i < top; i++) rest |= m[i];
    const uint32_t t = m[top] ^ (1u << ((bl - 1) & 31));
    rest |= top == 0 ? t >> 1 : (t | (m[0] >> 1));
    return rest ? bl : bl - 1;
}
// one candidate of `bits` bits into out[0 .. limbs)
__device__ __forceinline__ void attempt(Stream& s, uint32_t* out, int limbs, int bits) {
    const int words = (bits + 31) >> 5;
    for (int w = 0; w < words; w += 16)
        chacha::block_to(out + w, words - w < 16 ? words - w : 16, s.key, s.counter++, s.stream, s.id_lo, s.id_hi);
    if (bits & 31) out[words - 1] &= (1u << (bits & 31)) - 1u;
    for (int i = words; i < limbs; i++) out[i] = 0;
    s.attempts++;
}
// gcd(v, m) == 1 for v < m < 2^(32 nm), m > 1: subtract-and-shift binary GCD on two thread-private copies (the candidate itself
// stays in the output row).  Both arrays are filled and consumed inside this one function (DESIGN section 9, toolchain note).
__device__ __forceinline__ bool coprime(const uint32_t* v, const uint32_t* m, int nm) {
    uint32_t A[MAX_LIMBS], B[MAX_LIMBS];
    int n = nm;
    while (n > 1 && m[n - 1] == 0) n--;
    for (int i = 0; i < n; i++) { A[i] = v[i]; B[i] = m[i]; }
    if (((A[0] | B[0]) & 1u) == 0) return false;         // both even (covers v = 0 under an even m)
    uint32_t *x = A, *y = B;                              // invariant: y odd, gcd(x, y) = gcd(v, m)
    if ((B[0] & 1u) == 0) { x = B; y = A; }
    for (;;) {
        while (n > 1 && (x[n - 1] | y[n - 1]) == 0) n--;
        if (st::is_zero(x, n)) break;
        while (x[0] == 0) {                               // x != 0: ends
            for (int i = 0; i + 1 < n; i++) x[i] = x[i + 1];
            x[n - 1] = 0;
        }
        const int tz = 31 - __clz(x[0] & (0u - x[0]));
        if (tz) {
            for (int i = 0; i + 1 < n; i++) x[i] = (x[i] >> tz) | (x[i + 1] << (32 - tz));
            x[n - 1] >>= tz;
        }
        if (st::cmp(x, y, n) < 0) { uint32_t* t = x; x = y; y = t; }
        st::sub(x, x, y, n);                              // odd - odd: even or zero
    }
    uint32_t hi = 0;
    for (int i = 1; i < n; i++) hi |= y[i];
    return y[0] == 1u && hi == 0;
}

// One value of `kind` into out[0 .. limbs).  bound = nb limbs (ignored for BITS and SCALAR), bits = the width of BITS.
// false (and out zeroed) for a degenerate request — bound 0, bound 1 for UNIT, bound < 3 for RANGE1, a bound or a BITS width
// that does not fit `limbs`, limbs < 8 for SCALAR — and after `cap` rejected candidates.
__device__ __forceinline__ bool sample(Stream& s, int kind, uint32_t* out, int limbs, const uint32_t* bound, int nb, int bits, uint32_t cap) {
    int width = 0;
    bool ok = true;
    if (kind == TECDSA_SAMPLE_BITS) width = bits;
    else if (kind == TECDSA_SAMPLE_SCALAR) { bound = Q_LIMBS; nb = 8; width = 256; }
    else {
        const int bl = bit_length(bound, nb);
        const int least = kind == TECDSA_SAMPLE_BELOW ? 1 : 2;        // smallest accepted bit_length: bound >= 1 / >= 2
        ok = bl >= least && !(kind == TECDSA_SAMPLE_RANGE1 && bl == 2 && bound[0] == 2u);
        if (ok) width = kind == TECDSA_SAMPLE_RANGE1 ? bit_length_minus2(bound, nb) : bl;
    }
    ok = ok && width >= 1 && width <= 32 * limbs;
    while (ok && s.attempts < cap) {
        attempt(s, out, limbs, width);
        if (kind == TECDSA_SAMPLE_BITS) return true;
        if (kind == TECDSA_SAMPLE_RANGE1) {
            // v < bound - 2  <=>  v + 2 < bound; the value is 1 + v
            uint64_t c = 2;
            for (int i = 0; i < limbs && c; i++) { c += out[i]; out[i] = (uint32_t)c; c >>= 32; }
            if (c || st::cmp2(out, limbs, bound, nb) >= 0) continue;
            uint32_t brw = 1;
            for (int i = 0; i < limbs && brw; i++) { brw = out[i] == 0; out[i] -= 1u; }
            return true;
        }
        if (st::cmp2(out, limbs, bound, nb) >= 0) continue;
        if (kind == TECDSA_SAMPLE_SCALAR && st::is_zero(out, 8)) continue;
        if (kind == TECDSA_SAMPLE_UNIT && !coprime(out, bound, nb)) continue;
        return true;
    }
    st::zero(out, limbs);
    return false;
}

// ---- the randomness record of one GG20 offline unit (TECDSA_RND_*), one call per (unit, field) ------------------------------
// f = the field's stream id (TECDSA_RNDS_*).  own / peer = key rows of the unit and of its co-signer, row0 = key row of party 0
// of the unit's key set (statement x is row0 + x); n_tab = [rows][64] Paillier moduli; qnt = [rows][72] q N~, q3nt = [rows][88]
// q^3 N~ (gg20_sample_bounds).  Bounds and order of use follow `sample_unit` of oracle/sampling.py line by line.
__device__ __forceinline__ bool gg20_sample_field(const uint32_t* key, uint64_t unit_id, int f, uint32_t own, uint32_t peer, uint32_t row0,
                                                  const uint32_t* n_tab, const uint32_t* qnt, const uint32_t* q3nt, uint32_t* rec, uint32_t cap) {
    int kind = TECDSA_SAMPLE_SCALAR, off = 0, limbs = 8, nb = 0, bits = 0;
    const uint32_t* bound = nullptr;
    const uint32_t *n_own = n_tab + (size_t)own * 64, *n_peer = n_tab + (size_t)peer * 64;
    if (f >= TECDSA_RNDS_ALICE && f < TECDSA_RNDS_ALICE + 12) {
        const int x = (f - TECDSA_RNDS_ALICE) >> 2, part = (f - TECDSA_RNDS_ALICE) & 3;
        const size_t st_row = (size_t)row0 + x;
        off = TECDSA_RND_ALICE + x * TECDSA_RND_ALICE_STRIDE;
        kind = TECDSA_SAMPLE_BELOW;
        if (part == 0) { off += TECDSA_RND_ALICE_ALPHA; limbs = 24; bound = Q3_LIMBS; nb = 24; }
        else if (part == 1) { off += TECDSA_RND_ALICE_BETA; limbs = 64; bound = n_own; nb = 64; kind = TECDSA_SAMPLE_UNIT; }
        else if (part == 2) { off += TECDSA_RND_ALICE_GAMMA; limbs = 88; bound = q3nt + st_row * 88; nb = 88; }
        else { off += TECDSA_RND_ALICE_RHO; limbs = 72; bound = qnt + st_row * 72; nb = 72; }
    } else {
        switch (f) {
        case TECDSA_RNDS_GAMMA: off = TECDSA_RND_GAMMA; break;
        case TECDSA_RNDS_K: off = TECDSA_RND_K; break;
        case TECDSA_RNDS_BLIND: off = TECDSA_RND_BLIND; kind = TECDSA_SAMPLE_BITS; bits = 256; break;
        case TECDSA_RNDS_RK: off = TECDSA_RND_RK; kind = TECDSA_SAMPLE_BELOW; limbs = 64; bound = n_own; nb = 64; break;
        case TECDSA_RNDS_BETATAG_GAMMA: off = TECDSA_RND_BETATAG_GAMMA; kind = TECDSA_SAMPLE_BELOW; limbs = 64; bound = n_peer; nb = 64; break;
        case TECDSA_RNDS_R_GAMMA: off = TECDSA_RND_R_GAMMA; kind = TECDSA_SAMPLE_BELOW; limbs = 64; bound = n_peer; nb = 64; break;
        case TECDSA_RNDS_NONCE_GAMMA_B: off = TECDSA_RND_NONCE_GAMMA_B; break;
        case TECDSA_RNDS_NONCE_GAMMA_BETA: off = TECDSA_RND_NONCE_GAMMA_BETA; break;
        case TECDSA_RNDS_BETATAG_W: off = TECDSA_RND_BETATAG_W; kind = TECDSA_SAMPLE_BELOW; limbs = 64; bound = n_peer; nb = 64; break;
        case TECDSA_RNDS_R_W: off = TECDSA_RND_R_W; kind = TECDSA_SAMPLE_BELOW; limbs = 64; bound = n_peer; nb = 64; break;
        case TECDSA_RNDS_NONCE_W_B: off = TECDSA_RND_NONCE_W_B; break;
        case TECDSA_RNDS_NONCE_W_BETA: off = TECDSA_RND_NONCE_W_BETA; break;
        case TECDSA_RNDS_L: off = TECDSA_RND_L; break;
        case TECDSA_RNDS_PED_S1: off = TECDSA_RND_PED_S1; break;
        case TECDSA_RNDS_PED_S2: off = TECDSA_RND_PED_S2; break;
        // PDLwSlackProof::prove against the PEER's (h1, h2, N~), beta under the prover's own Paillier key
        case TECDSA_RNDS_PDL_ALPHA: off = TECDSA_RND_PDL_ALPHA; kind = TECDSA_SAMPLE_BELOW; limbs = 24; bound = Q3_LIMBS; nb = 24; break;
        case TECDSA_RNDS_PDL_BETA: off = TECDSA_RND_PDL_BETA; kind = TECDSA_SAMPLE_RANGE1; limbs = 64; bound = n_own; nb = 64; break;
        case TECDSA_RNDS_PDL_RHO: off = TECDSA_RND_PDL_RHO; kind = TECDSA_SAMPLE_BELOW; limbs = 72; bound = qnt + (size_t)peer * 72; nb = 72; break;
        case TECDSA_RNDS_PDL_GAMMA: off = TECDSA_RND_PDL_GAMMA; kind = TECDSA_SAMPLE_BELOW; limbs = 88; bound = q3nt + (size_t)peer * 88; nb = 88; break;
        case TECDSA_RNDS_HEG_S1: off = TECDSA_RND_HEG_S1; break;
        case TECDSA_RNDS_HEG_S2: off = TECDSA_RND_HEG_S2; break;
        default: return false;
        }
    }
    Stream s = open(key, (uint32_t)f, unit_id);
    return sample(s, kind, rec + off, limbs, bound, nb, bits, cap);
}
// row r of qnt (72 limbs) = q N~_r for which = 0, of q3nt (88 limbs) = q^3 N~_r for which = 1
__device__ __forceinline__ void gg20_sample_bounds(const uint32_t* nt_tab, uint32_t* qnt, uint32_t* q3nt, int r, int which) {
    const uint32_t* nt = nt_tab + (size_t)r * 64;
    if (which == 0) st::mul_add(qnt + (size_t)r * 72, 72, Q_LIMBS, 8, nt, 64, nullptr, 0);
    else st::mul_add(q3nt + (size_t)r * 88, 88, Q3_LIMBS, 24, nt, 64, nullptr, 0);
}

}  // namespace smp
}  // namespace tecdsa
