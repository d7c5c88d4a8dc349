// Seeded sampling entry points (include/tecdsa_b200.h, "seeded sampling"): the values the reference draws from the OS RNG inside
// `MessageA::a`, `MessageB::b`, `AliceProof::generate`, `PDLwSlackProof::prove`, `SignKeys::create` (/root/reference/src/utilities/
// mta/mod.rs:57,97-98, mta/range_proofs.rs:48-51,538-557, zk_pdl_with_slack/mod.rs:73-77, protocols/multi_party_ecdsa/gg_2020/
// party_i.rs:563-574,628), derived on the device from one caller-supplied seed.  Rules and keystream layout: sampler.cuh.
#include "sampler.cuh"
#include "stage.cuh"

using namespace tecdsa;

namespace {

// L0: one thread per element
__global__ void __launch_bounds__(128) k_sample(const uint32_t* seed, uint64_t first_id, uint32_t stream, int kind, int bits, const uint32_t* bound,
                                                const uint32_t* idx, uint32_t n_bound, int limbs, uint32_t* out, uint8_t* status, int count) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    uint32_t* o = out + (size_t)i * limbs;
    const uint32_t row = idx ? idx[i] : (uint32_t)i;
    bool ok = !bound || !idx || row < n_bound;
    if (ok) {
        smp::Stream s = smp::open(seed, stream, first_id + (uint64_t)i);
        ok = smp::sample(s, kind, o, limbs, bound ? bound + (size_t)row * limbs : nullptr, limbs, bits, TECDSA_SAMPLE_ATTEMPTS);
    } else st::zero(o, limbs);
    status[i] = ok ? TECDSA_ST_OK : TECDSA_ST_SAMPLING;
}
__global__ void k_gg20_sample_bounds(const uint32_t* nt_tab, uint32_t* qnt, uint32_t* q3nt, int rows) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t < 2 * rows) smp::gg20_sample_bounds(nt_tab, qnt, q3nt, t % rows, t / rows);
}
// L3: one thread per (field, unit), field-major: the lanes of a warp draw the same field of 32 units, so the warps of the three
// coprimality tests per unit are full and every other warp never enters one.  status is zeroed before the launch.
__global__ void __launch_bounds__(128) k_gg20_sample(const uint32_t* seed, uint64_t first_unit, const uint32_t* sessions, uint32_t n_keysets,
                                                     const uint32_t* n_tab, const uint32_t* qnt, const uint32_t* q3nt, uint32_t* rnd, uint8_t* status, int U) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= U * TECDSA_RNDS_COUNT) return;
    const int u = t % U;
    const int f = t / U;                    // the field's stream id: TECDSA_RNDS_* are 0 .. TECDSA_RNDS_COUNT - 1 without gaps
    const uint32_t* d = sessions + (size_t)(u >> 1) * 3;
    const uint32_t ks = d[0], own = d[1 + (u & 1)], peer = d[2 - (u & 1)];
    uint32_t* rec = rnd + (size_t)u * TECDSA_RND_LIMBS;
    if (ks >= n_keysets || own > 2 || peer > 2 || own == peer) {
        if (f == 0) { st::zero(rec, TECDSA_RND_LIMBS); status[u] = TECDSA_ST_SAMPLING; }
        return;
    }
    if (!smp::gg20_sample_field(seed, first_unit + (uint64_t)u, f, ks * 3 + own, ks * 3 + peer, ks * 3, n_tab, qnt, q3nt, rec, TECDSA_SAMPLE_ATTEMPTS))
        status[u] = TECDSA_ST_SAMPLING;
}

// the seed is a secret of the grade of the nonces: it travels through wiped device scratch, never as a kernel argument
const uint32_t* stage_seed(Stage& S, const uint32_t* seed) {
    uint32_t* d = S.tmp<uint32_t>(8);
    if (d && cudaMemcpyAsync(d, seed, 32, cudaMemcpyHostToDevice, S.c->stream) != cudaSuccess) S.err = tecdsa_fail(TECDSA_E_CUDA, "H2D copy of the seed");
    return d;
}

}  // namespace

extern "C" int tecdsa_sample_batch(tecdsa_ctx* c, const uint32_t seed[8], uint64_t first_id, uint32_t stream, int kind, int bits, const uint32_t* bound,
                                   const uint32_t* bound_idx, size_t n_bound, int limbs, uint32_t* out, uint8_t* status, size_t count, int mem) {
    if (!seed || !out || !status) return tecdsa_fail(TECDSA_E_ARG, "sample: null argument");
    if (kind < TECDSA_SAMPLE_BITS || kind > TECDSA_SAMPLE_SCALAR) return tecdsa_fail(TECDSA_E_ARG, "sample: unknown kind");
    if (limbs < 1 || limbs > TECDSA_SAMPLE_MAX_LIMBS) return tecdsa_fail(TECDSA_E_ARG, "sample: limbs must be 1..128");
    const bool bounded = kind == TECDSA_SAMPLE_BELOW || kind == TECDSA_SAMPLE_UNIT || kind == TECDSA_SAMPLE_RANGE1;
    if (bounded && (!bound || (bound_idx && n_bound == 0))) return tecdsa_fail(TECDSA_E_ARG, "sample: this kind needs a bound table");
    if (kind == TECDSA_SAMPLE_BITS && (bits < 1 || bits > 32 * limbs)) return tecdsa_fail(TECDSA_E_ARG, "sample: bits must be 1..32*limbs");
    if (kind == TECDSA_SAMPLE_SCALAR && limbs < 8) return tecdsa_fail(TECDSA_E_ARG, "sample: a scalar needs 8 limbs");
    if (count > (1u << 30) || n_bound > 0xFFFFFFFFu) return tecdsa_fail(TECDSA_E_ARG, "sample: too many elements");
    STAGE_PROLOGUE("sample", count);
    const uint32_t* dseed = stage_seed(S, seed);
    const uint32_t* db = bounded ? S.in(bound, (bound_idx ? n_bound : count) * (size_t)limbs) : nullptr;
    const uint32_t* di = bounded ? S.in(bound_idx, count) : nullptr;
    uint32_t* dout = S.out(out, count * (size_t)limbs);
    uint8_t* dst = S.out(status, count);
    if (S.err) return S.err;
    c->prof_begin("sample");
    k_sample<<<(unsigned)((count + 127) / 128), 128, 0, c->stream>>>(dseed, first_id, stream, kind, bits, db, di, (uint32_t)n_bound, limbs, dout, dst, (int)count);
    c->prof_end();
    KCHECK();
    return S.finish();
}

extern "C" int tecdsa_gg20_sample_randomness(tecdsa_ctx* c, const tecdsa_keyset* ks, const uint32_t* sessions, size_t n_sessions, const uint32_t seed[8],
                                             uint64_t first_unit, uint32_t* rnd, uint8_t* status, int mem) {
    if (!ks || !sessions || !seed || !rnd || !status) return tecdsa_fail(TECDSA_E_ARG, "gg20_sample_randomness: null argument");
    if (ks->parties != 3) return tecdsa_fail(TECDSA_E_ARG, "gg20_sample_randomness: the key set must have three parties");
    if (n_sessions > (1u << 22)) return tecdsa_fail(TECDSA_E_ARG, "gg20_sample_randomness: too many sessions");
    STAGE_PROLOGUE("gg20_sample_randomness", n_sessions);
    const size_t U = 2 * n_sessions;
    const int rows = ks->n_keysets * 3;
    const uint32_t* dseed = stage_seed(S, seed);
    const uint32_t* dsess = S.in(sessions, n_sessions * 3);
    uint32_t* drnd = S.out(rnd, U * TECDSA_RND_LIMBS);
    uint8_t* dst = S.out(status, U);
    uint32_t *qnt = S.tmp<uint32_t>((size_t)rows * 72), *q3nt = S.tmp<uint32_t>((size_t)rows * 88);
    if (S.err) return S.err;
    CK(cudaMemsetAsync(dst, 0, U, c->stream));
    k_gg20_sample_bounds<<<(2 * rows + 63) / 64, 64, 0, c->stream>>>(ks->tab[KT_NT], qnt, q3nt, rows);
    KCHECK();
    c->prof_begin("gg20_sample");
    k_gg20_sample<<<(unsigned)((U * TECDSA_RNDS_COUNT + 127) / 128), 128, 0, c->stream>>>(dseed, first_unit, dsess, (uint32_t)ks->n_keysets, ks->tab[KT_N], qnt, q3nt,
                                                                                         drnd, dst, (int)U);
    c->prof_end();
    KCHECK();
    return S.finish();
}
