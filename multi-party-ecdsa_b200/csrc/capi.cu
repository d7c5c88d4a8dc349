// C ABI of the engine (see include/tecdsa_b200.h).  Host side: context, workspace,
// staging of host buffers, launch geometry.  No torch types, no CPU arithmetic fallback:
// if CUDA is unavailable every entry point fails with TECDSA_E_CUDA.
#include "ctx.h"
#include "modinv.cuh"
#include "nadic.cuh"
#include "nadic_inv.cuh"

#include <cstdio>
#include <cstdlib>
#include <string>

using namespace tecdsa;

static thread_local std::string g_err;
int tecdsa_fail(int code, const char* what, cudaError_t e) {
    g_err = what;
    if (e != cudaSuccess) { g_err += ": "; g_err += cudaGetErrorString(e); }
    return code;
}
static int fail(int code, const char* what, cudaError_t e = cudaSuccess) { return tecdsa_fail(code, what, e); }

static int ws_reserve(tecdsa_ctx* c, size_t bytes) {
    if (bytes <= c->ws_bytes) return 0;
    CK(cudaStreamSynchronize(c->stream));
    if (c->ws) CK(cudaFree(c->ws));
    c->ws = nullptr; c->ws_bytes = 0;
    size_t want = bytes + (bytes >> 3);
    cudaError_t e = cudaMalloc(&c->ws, want);
    if (e != cudaSuccess) { want = bytes; e = cudaMalloc(&c->ws, want); }
    if (e != cudaSuccess) return fail(TECDSA_E_NOMEM, "cudaMalloc(workspace)", e);
    c->ws_bytes = want;
    return 0;
}
struct Bump {
    char* p; size_t off = 0;
    explicit Bump(char* base) : p(base) {}
    template <typename T> T* take(size_t n) {
        off = (off + 255) & ~size_t(255);
        T* r = reinterpret_cast<T*>(p + off);
        off += n * sizeof(T);
        return r;
    }
};
static size_t al(size_t x) { return (x + 255) & ~size_t(255); }
static bool default_sqr();

extern "C" int tecdsa_ctx_create(tecdsa_ctx** out, int device, void* stream) {
    if (!out) return fail(TECDSA_E_ARG, "ctx_create: null out");
    int ndev = 0;
    CK(cudaGetDeviceCount(&ndev));
    if (device < 0 || device >= ndev) return fail(TECDSA_E_ARG, "ctx_create: bad device");
    CK(cudaSetDevice(device));
    tecdsa_ctx* c = new tecdsa_ctx();
    c->device = device;
    c->stream = (cudaStream_t)stream;              // NULL = the device's default stream
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, device));
    c->sm_count = prop.multiProcessorCount;
    c->opt_sqr = default_sqr();
    // the glue kernels call non-inlined EC / hash routines with multi-KB frames
    CK(cudaDeviceSetLimit(cudaLimitStackSize, 16 * 1024));
    {
        const uint32_t* fbp = nullptr;
        int rc = tecdsa_internal_fb_points_init(device, c->stream, &fbp);
        if (rc == 0) rc = tecdsa_internal_fb_points_set_l12(fbp);
        if (rc == 0) rc = tecdsa_internal_fb_points_set_keygen(fbp);
        if (rc == 0) rc = tecdsa_internal_fb_points_set_records(fbp);
        if (rc == 0) rc = tecdsa_internal_fb_points_set_ecops(fbp);
        if (rc == 0) rc = tecdsa_internal_fb_points_set_blame(fbp);
        if (rc == 0) rc = tecdsa_internal_fb_points_set_lindell17(fbp);
        if (rc == 0) rc = tecdsa_internal_fb_points_set_gg18(fbp);
        if (rc) { delete c; return rc; }
    }
    CK(cudaEventCreate(&c->ev0));
    CK(cudaEventCreate(&c->ev1));
    CK(cudaMalloc(&c->d_work, sizeof(unsigned long long)));
    CK(cudaMemsetAsync(c->d_work, 0, sizeof(unsigned long long), c->stream));
    *out = c;
    return 0;
}
extern "C" int tecdsa_ctx_destroy(tecdsa_ctx* c) {
    if (!c) return 0;
    cudaSetDevice(c->device);
    cudaStreamSynchronize(c->stream);
    for (int h = 0; h < 2; h++) {
        if (c->child[h]) tecdsa_ctx_destroy(c->child[h]);
        if (c->ev_join[h]) cudaEventDestroy(c->ev_join[h]);
    }
    if (c->ev_fork) cudaEventDestroy(c->ev_fork);
    // secrets may sit in every scratch buffer: wipe before release (the reference zeroizes its
    // proof round-1 secrets on drop, utilities/mta/range_proofs.rs:26-27)
    char* bufs[4] = {c->ws, c->jobmem, c->arena, c->rec};
    size_t sizes[4] = {c->ws_bytes, c->jobmem_bytes, c->arena_bytes, c->rec_bytes};
    for (int i = 0; i < 4; i++) if (bufs[i]) cudaMemsetAsync(bufs[i], 0, sizes[i], c->stream);
    cudaStreamSynchronize(c->stream);
    for (int i = 0; i < 4; i++) if (bufs[i]) cudaFree(bufs[i]);
    if (c->d_work) cudaFree(c->d_work);
    cudaEventDestroy(c->ev0); cudaEventDestroy(c->ev1);
    if (c->owns_stream) cudaStreamDestroy(c->stream);
    delete c;
    return 0;
}
extern "C" int tecdsa_ctx_sync(tecdsa_ctx* c) {
    if (!c) return fail(TECDSA_E_ARG, "null ctx");
    CK(cudaStreamSynchronize(c->stream));
    return 0;
}
extern "C" const char* tecdsa_last_error(void) { return g_err.c_str(); }
extern "C" int tecdsa_ctx_set_tpi(tecdsa_ctx* c, int mod_bits, int tpi) {
    if (!c) return fail(TECDSA_E_ARG, "null ctx");
    int slot = mod_bits == 1024 ? 0 : mod_bits == 2048 ? 1 : mod_bits == 4096 ? 2 : -1;
    if (slot < 0) return fail(TECDSA_E_ARG, "set_tpi: mod_bits must be 1024/2048/4096");
    if (tpi != 0 && tpi != 4 && tpi != 8 && tpi != 16 && tpi != 32) return fail(TECDSA_E_ARG, "set_tpi: tpi must be 0/4/8/16/32");
    c->tpi[slot] = tpi;
    return 0;
}
extern "C" int tecdsa_ctx_set_option(tecdsa_ctx* c, const char* name, int value) {
    if (!c || !name) return fail(TECDSA_E_ARG, "ctx_set_option: null argument");
    if (strcmp(name, "sqr") == 0) { c->opt_sqr = value != 0; return 0; }
    return fail(TECDSA_E_ARG, "ctx_set_option: unknown option");
}
extern "C" int tecdsa_ctx_last_kernel_ms(tecdsa_ctx* c, float* ms, int* launches) {
    if (!c) return fail(TECDSA_E_ARG, "null ctx");
    CK(cudaEventSynchronize(c->ev1));
    float t = 0.f;
    CK(cudaEventElapsedTime(&t, c->ev0, c->ev1));
    c->last_ms = t;
    if (ms) *ms = t;
    if (launches) *launches = c->last_launches;
    return 0;
}
extern "C" uint64_t tecdsa_ctx_launch_count(tecdsa_ctx* c) { return c ? c->launches : 0; }

// ------------------------------------------------------------------------------------ per-launch profiling
void tecdsa_ctx::prof_begin(const char* name) {
    if (!profiling || prof.size() >= prof_cap) return;
    ProfEntry e{name, nullptr, nullptr};
    if (cudaEventCreate(&e.e0) != cudaSuccess || cudaEventCreate(&e.e1) != cudaSuccess) return;
    cudaEventRecord(e.e0, stream);
    prof.push_back(e);
}
void tecdsa_ctx::prof_end() {
    if (!profiling || prof.empty() || prof.size() > prof_cap) return;
    cudaEventRecord(prof.back().e1, stream);
    cudaMemcpyAsync(prof_work + prof.size() - 1, d_work, sizeof(unsigned long long), cudaMemcpyDeviceToHost, stream);
}
extern "C" int tecdsa_ctx_profile(tecdsa_ctx* c, int enable) {
    if (!c) return fail(TECDSA_E_ARG, "ctx_profile: null ctx");
    CK(cudaSetDevice(c->device));
    CK(cudaStreamSynchronize(c->stream));
    for (auto& e : c->prof) { cudaEventDestroy(e.e0); cudaEventDestroy(e.e1); }
    c->prof.clear();
    if (enable && !c->prof_work) {
        c->prof_cap = 4096;
        CK(cudaMallocHost(&c->prof_work, c->prof_cap * sizeof(unsigned long long)));
    }
    if (enable) {
        CK(cudaMemcpyAsync(&c->prof_work_base, c->d_work, sizeof(unsigned long long), cudaMemcpyDeviceToHost, c->stream));
        CK(cudaStreamSynchronize(c->stream));
    }
    c->profiling = enable != 0;
    return 0;
}
extern "C" int tecdsa_ctx_profile_read(tecdsa_ctx* c, tecdsa_launch_info* out, size_t cap, size_t* n) {
    if (!c || !n) return fail(TECDSA_E_ARG, "ctx_profile_read: null argument");
    CK(cudaSetDevice(c->device));
    CK(cudaStreamSynchronize(c->stream));
    *n = c->prof.size();
    unsigned long long prev = 0;
    for (size_t i = 0; i < c->prof.size() && out && i < cap; i++) {
        float ms = 0.f;
        CK(cudaEventElapsedTime(&ms, c->prof[i].e0, c->prof[i].e1));
        memset(&out[i], 0, sizeof(out[i]));
        strncpy(out[i].kernel, c->prof[i].name, sizeof(out[i].kernel) - 1);
        out[i].ms = ms;
        out[i].mac32 = i == 0 ? 0 : c->prof_work[i] - prev;
        if (i == 0) out[i].mac32 = c->prof_work[0] - c->prof_work_base;
        prev = c->prof_work[i];
    }
    return 0;
}

// ------------------------------------------------------------------------------------ modexp
// Squarings of tecdsa_modexp_batch through the block-partitioned mont_sqr (sqr.cuh) instead of mont_mul(a, a): bit-identical,
// 12.5-19 % fewer multiply-accumulates, but MEASURED SLOWER on an H100 at 400 W (2048-bit, 65 536 operands: 344 ms vs 187 ms
// with 4 lanes, 279 vs 203 ms with 8) — the shuffles and in-lane accumulation that re-balance the triangle across
// lock-stepped lanes cost more issue slots than the saved IMAD.WIDE pipe time.  Kept selectable (tecdsa_ctx_set_option "sqr",
// TECDSA_SQR=1) so that the parity test covers it and the measurement can be repeated; off by default.
static bool default_sqr() {
    static const bool on = [] { const char* e = getenv("TECDSA_SQR"); return e && atoi(e) != 0; }();
    return on;
}
// One block per 128/TPI operands, window table per operand.
template <int K, int TPI>
static cudaError_t launch_modexp(bool sqr, cudaStream_t s, const uint32_t* base, const uint32_t* exp, const uint32_t* mod,
                                 const uint32_t* mod_idx, uint32_t* out, uint8_t* status, uint32_t* table,
                                 int count, int exp_limbs, unsigned long long* work) {
    constexpr int BLOCK = 128;
    constexpr int PER_BLOCK = BLOCK / TPI;
    int grid = (count + PER_BLOCK - 1) / PER_BLOCK;
    if (sqr) modexp_kernel<K, TPI, true><<<grid, BLOCK, 0, s>>>(base, exp, mod, mod_idx, out, status, table, count, exp_limbs, work);
    else modexp_kernel<K, TPI, false><<<grid, BLOCK, 0, s>>>(base, exp, mod, mod_idx, out, status, table, count, exp_limbs, work);
    return cudaGetLastError();
}

// kernel time on an H100 at 400 W, 2048-bit exponents: 65 536 x 2048-bit 187 / 203 ms for TPI 4 / 8; 65 536 x 1024-bit 52 / 64 ms
// for TPI 4 / 8; 16 384 x 4096-bit 186 / 203 ms for TPI 8 / 16
static int default_tpi(int mod_bits) { return mod_bits == 1024 ? 4 : mod_bits == 2048 ? 4 : 8; }

static cudaError_t dispatch_modexp(bool sqr, int mod_bits, int tpi, cudaStream_t s, const uint32_t* base, const uint32_t* exp,
                                   const uint32_t* mod, const uint32_t* mod_idx, uint32_t* out, uint8_t* status,
                                   uint32_t* table, int count, int exp_limbs, unsigned long long* work) {
#define GO(K, T) return launch_modexp<K, T>(sqr, s, base, exp, mod, mod_idx, out, status, table, count, exp_limbs, work)
    switch (mod_bits) {
    case 1024: switch (tpi) { case 4: GO(32, 4); case 8: GO(32, 8); case 16: GO(32, 16); default: return cudaErrorInvalidValue; }
    case 2048: switch (tpi) { case 4: GO(64, 4); case 8: GO(64, 8); case 16: GO(64, 16); case 32: GO(64, 32); default: return cudaErrorInvalidValue; }
    case 4096: switch (tpi) { case 8: GO(128, 8); case 16: GO(128, 16); case 32: GO(128, 32); default: return cudaErrorInvalidValue; }
    }
#undef GO
    return cudaErrorInvalidValue;
}

extern "C" int tecdsa_modexp_batch(tecdsa_ctx* c, int mod_bits, int exp_limbs, const uint32_t* base, const uint32_t* exp,
                                   const uint32_t* modulus, const uint32_t* mod_idx, size_t n_mod, uint32_t* out,
                                   uint8_t* status, size_t count, int mem) {
    if (!c) return fail(TECDSA_E_ARG, "null ctx");
    if (mod_bits != 1024 && mod_bits != 2048 && mod_bits != 4096) return fail(TECDSA_E_UNSUPPORTED, "modexp: mod_bits must be 1024/2048/4096");
    if (exp_limbs <= 0 || exp_limbs > 4096) return fail(TECDSA_E_ARG, "modexp: exp_limbs out of range");
    if (count == 0) { c->last_launches = 0; return 0; }
    if (!base || !exp || !modulus || !out) return fail(TECDSA_E_ARG, "modexp: null buffer");
    if (mem != TECDSA_HOST && mem != TECDSA_DEVICE) return fail(TECDSA_E_ARG, "modexp: bad mem");
    if (count > (size_t)1 << 30) return fail(TECDSA_E_ARG, "modexp: count too large");
    CK(cudaSetDevice(c->device));
    const int K = mod_bits / 32;
    const int slot = mod_bits == 1024 ? 0 : mod_bits == 2048 ? 1 : 2;
    const int tpi = c->tpi[slot] ? c->tpi[slot] : default_tpi(mod_bits);
    if (!mod_idx) n_mod = count;
    if (n_mod == 0) return fail(TECDSA_E_ARG, "modexp: n_mod == 0");

    const size_t CHUNK = 1 << 17;                                // operands per launch (bounds the table)
    const size_t chunk = count < CHUNK ? count : CHUNK;
    const size_t per_block = 128 / tpi;
    const size_t slots = ((chunk + per_block - 1) / per_block) * per_block;
    const size_t table_words = slots * ((size_t)K << WINDOW_BITS);
    size_t need = al(table_words * 4);
    if (mem == TECDSA_HOST)
        need += al(chunk * K * 4) * 2 + al(chunk * exp_limbs * 4) + al(n_mod * K * 4) + al(chunk * 4) + al(chunk) + 4096;
    int rc = ws_reserve(c, need);
    if (rc) return rc;
    Bump bump(c->ws);
    uint32_t* d_table = bump.take<uint32_t>(table_words);
    uint32_t *d_base = nullptr, *d_exp = nullptr, *d_mod = nullptr, *d_idx = nullptr, *d_out = nullptr;
    uint8_t* d_status = nullptr;
    if (mem == TECDSA_HOST) {
        d_base = bump.take<uint32_t>(chunk * K);
        d_out = bump.take<uint32_t>(chunk * K);
        d_exp = bump.take<uint32_t>(chunk * exp_limbs);
        d_mod = bump.take<uint32_t>(n_mod * K);
        d_idx = bump.take<uint32_t>(chunk);
        d_status = bump.take<uint8_t>(chunk);
        if (mod_idx) CK(cudaMemcpyAsync(d_mod, modulus, n_mod * K * 4, cudaMemcpyHostToDevice, c->stream));
    }
    int launches = 0;
    bool first = true;
    for (size_t off = 0; off < count; off += chunk) {
        const size_t m = (count - off < chunk) ? count - off : chunk;
        const uint32_t *kb, *ke, *km, *ki; uint32_t* ko; uint8_t* ks;
        if (mem == TECDSA_HOST) {
            CK(cudaMemcpyAsync(d_base, base + off * K, m * K * 4, cudaMemcpyHostToDevice, c->stream));
            CK(cudaMemcpyAsync(d_exp, exp + off * exp_limbs, m * exp_limbs * 4, cudaMemcpyHostToDevice, c->stream));
            if (mod_idx) CK(cudaMemcpyAsync(d_idx, mod_idx + off, m * 4, cudaMemcpyHostToDevice, c->stream));
            else CK(cudaMemcpyAsync(d_mod, modulus + off * K, m * K * 4, cudaMemcpyHostToDevice, c->stream));
            kb = d_base; ke = d_exp; km = d_mod; ki = mod_idx ? d_idx : nullptr; ko = d_out; ks = status ? d_status : nullptr;
        } else {
            kb = base + off * K; ke = exp + off * exp_limbs; km = mod_idx ? modulus : modulus + off * K;
            ki = mod_idx ? mod_idx + off : nullptr; ko = out + off * K; ks = status ? status + off : nullptr;
        }
        if (first) { CK(cudaEventRecord(c->ev0, c->stream)); first = false; }
        c->prof_begin("modexp_kernel");
        cudaError_t e = dispatch_modexp(c->opt_sqr, mod_bits, tpi, c->stream, kb, ke, km, ki, ko, ks, d_table, (int)m, exp_limbs, c->d_work);
        c->prof_end();
        if (e != cudaSuccess) return fail(e == cudaErrorInvalidValue ? TECDSA_E_UNSUPPORTED : TECDSA_E_CUDA, "modexp launch", e);
        launches++;
        CK(cudaEventRecord(c->ev1, c->stream));
        if (mem == TECDSA_HOST) {
            CK(cudaMemcpyAsync(out + off * K, d_out, m * K * 4, cudaMemcpyDeviceToHost, c->stream));
            if (status) CK(cudaMemcpyAsync(status + off, d_status, m, cudaMemcpyDeviceToHost, c->stream));
            if (off + chunk < count) CK(cudaStreamSynchronize(c->stream));   // staging buffers are reused
        }
    }
    c->last_launches = launches;
    c->launches += launches;
    if (mem == TECDSA_HOST) CK(cudaStreamSynchronize(c->stream));
    return 0;
}

// ------------------------------------------------------------------------------------ IMAD peak
// Saturation micro-benchmarks of the integer multiply-add pipe — the roofline denominators (SURVEY.md section 8d).
//  * carry-free: 16 independent 64-bit accumulators per thread, acc_j += a_j * b_u as IMAD.WIDE.U32 — every product of an
//    iteration has its OWN operand pair (16 distinct a_j, a fresh b_u per step), so ptxas cannot share a product between two
//    accumulators (the round-1 kernel reused operand pairs and ptxas turned half of its MACs into adds);
//  * carry-chained: the instruction the Montgomery rows are made of, IMAD.WIDE.U32.X with carry in and out — the mad_even /
//    mad_odd chains of bigint.cuh on two accumulator sets, exactly as mont_row issues them.
// Both run at full occupancy with few registers; tools/sass_mix.py prints the SASS mix of the two loops.
__global__ void __launch_bounds__(256) imad_peak_kernel(uint32_t* sink, uint32_t seed, int iters) {
    constexpr int NACC = 16;
    uint32_t acc[2 * NACC], a[NACC];                 // accumulator j = the register pair (acc[2j], acc[2j+1])
#pragma unroll
    for (int j = 0; j < NACC; j++) { a[j] = (seed + 0x9e3779b9u * (j + 1)) ^ (threadIdx.x * 2654435761u); acc[2 * j] = seed * (j + 1) + threadIdx.x; acc[2 * j + 1] = seed ^ j; }
    uint32_t b = seed ^ 0x85ebca6bu ^ threadIdx.x;
    // every multiply-accumulate is written as the lo/hi pair the Montgomery rows use (mad.lo.cc / madc.hi on neighbouring array
    // elements): the accumulator sits on an aligned register pair and the pair fuses into ONE IMAD.WIDE.U32 with accumulate; the
    // carry-flag dependence inside each pair also keeps ptxas from re-associating two products of one accumulator into two
    // multiplies and a three-input add (what it does to plain 64-bit mad.wide sequences)
#pragma unroll 1
    for (int it = 0; it < iters; it++) {
#pragma unroll
        for (int u = 0; u < 4; u++) {
#pragma unroll
            for (int j = 0; j < NACC; j++)
                asm volatile("mad.lo.cc.u32 %0, %2, %3, %0; madc.hi.u32 %1, %2, %3, %1;" : "+r"(acc[2 * j]), "+r"(acc[2 * j + 1]) : "r"(a[j]), "r"(b));
            b += 0x01000193u;                                            // a fresh multiplier per step
        }
    }
    uint32_t x = 0;
#pragma unroll
    for (int j = 0; j < 2 * NACC; j++) x ^= acc[j];
    if (x == 0x12345678u) sink[0] = x;
}
__global__ void __launch_bounds__(256) imad_chain_peak_kernel(uint32_t* sink, uint32_t seed, int iters) {
    constexpr int L = 16;
    uint32_t E[L + 2], O[L + 2], a[L];
#pragma unroll
    for (int j = 0; j < L; j++) a[j] = (seed + 0x9e3779b9u * (j + 1)) ^ (threadIdx.x * 2654435761u);
#pragma unroll
    for (int j = 0; j < L + 2; j++) { E[j] = seed + j; O[j] = seed ^ j; }
    uint32_t b = seed ^ 0x85ebca6bu ^ threadIdx.x;
#pragma unroll 1
    for (int it = 0; it < iters; it++) {
#pragma unroll
        for (int u = 0; u < 4; u++) {
            const uint32_t bu = b + 0x01000193u * (u + 1);
            mad_even<L>(E, a, bu);                                       // 8 IMAD.WIDE.U32(.X) in one carry chain
            mad_odd<L>(O, a, bu);                                        // 8 more on the second accumulator set
        }
        b = b * 5u + E[0];
    }
    uint32_t x = 0;
#pragma unroll
    for (int j = 0; j < L + 2; j++) x ^= E[j] ^ O[j];
    if (x == 0x12345678u) sink[0] = x;
}

static int imad_run(tecdsa_ctx* c, bool chained, double* mac32_per_s, float* ms_out) {
    CK(cudaSetDevice(c->device));
    int rc = ws_reserve(c, 4096);
    if (rc) return rc;
    const int iters = 1 << 13, block = 256, grid = c->sm_count * 16;
    const double macs_per_iter = chained ? 64.0 : 64.0;                   // 4 steps x 16 wide MACs per thread and iteration, both kernels
    float best = 1e30f;
    for (int rep = 0; rep < 4; rep++) {
        CK(cudaEventRecord(c->ev0, c->stream));
        if (chained) imad_chain_peak_kernel<<<grid, block, 0, c->stream>>>((uint32_t*)c->ws, 12345u + rep, rep ? iters : 64);
        else imad_peak_kernel<<<grid, block, 0, c->stream>>>((uint32_t*)c->ws, 12345u + rep, rep ? iters : 64);
        CK(cudaEventRecord(c->ev1, c->stream));
        CK(cudaEventSynchronize(c->ev1));
        float t;
        CK(cudaEventElapsedTime(&t, c->ev0, c->ev1));
        if (rep && t < best) best = t;                                   // rep 0 is the warm-up
    }
    CK(cudaGetLastError());
    c->launches += 4;
    if (mac32_per_s) *mac32_per_s = (double)grid * block * (double)iters * macs_per_iter / (best * 1e-3);
    if (ms_out) *ms_out = best;
    return 0;
}
extern "C" int tecdsa_imad_peak(tecdsa_ctx* c, double* mac32_per_s, float* ms_out) {
    if (!c) return fail(TECDSA_E_ARG, "null ctx");
    return imad_run(c, false, mac32_per_s, ms_out);
}
extern "C" int tecdsa_imad_peak_chained(tecdsa_ctx* c, double* mac32_per_s, float* ms_out) {
    if (!c) return fail(TECDSA_E_ARG, "null ctx");
    return imad_run(c, true, mac32_per_s, ms_out);
}

// ------------------------------------------------------------------------------------ job-list launches
static int grow(char** buf, size_t* have, size_t need, cudaStream_t s, const char* what) {
    if (need <= *have) return 0;
    CK(cudaStreamSynchronize(s));
    if (*buf) CK(cudaFree(*buf));
    *buf = nullptr; *have = 0;
    cudaError_t e = cudaMalloc(buf, need);
    if (e != cudaSuccess) return tecdsa_fail(TECDSA_E_NOMEM, what, e);
    *have = need;
    return 0;
}
int tecdsa_ctx::reserve_arena(size_t bytes) { return grow(&arena, &arena_bytes, bytes, stream, "cudaMalloc(arena)"); }

namespace {
constexpr int JOB_SLOTS = 64;
constexpr size_t SLOT_BYTES = (sizeof(ExpLaunch) + 255) & ~size_t(255);
constexpr int JOB_BLOCK = 128;
struct JobGeom { int grid; size_t table_bytes; };
template <int K, int TPI> JobGeom job_geom(int sm_count) {
    int per_sm = 0;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, exp_jobs_kernel<K, TPI>, JOB_BLOCK, 0);
    if (per_sm < 1) per_sm = 1;
    JobGeom g;
    g.grid = sm_count * per_sm;
    g.table_bytes = (size_t)g.grid * (JOB_BLOCK / 32) * (32 / TPI) * 2 * (size_t)(K << WINDOW_BITS) * 4;
    return g;
}
}  // namespace

static int job_prepare(tecdsa_ctx* c, size_t table_bytes, const void* desc, size_t desc_bytes, char** d_desc, unsigned int** d_counter, uint32_t** d_tables) {
    static_assert(sizeof(InvLaunch) <= sizeof(ExpLaunch), "slot size");
    const size_t head = JOB_SLOTS * SLOT_BYTES + JOB_SLOTS * 256;
    int rc = grow(&c->jobmem, &c->jobmem_bytes, head + table_bytes, c->stream, "cudaMalloc(job memory)");
    if (rc) return rc;
    if (c->job_slot == JOB_SLOTS) { CK(cudaStreamSynchronize(c->stream)); c->job_slot = 0; }
    const int slot = c->job_slot++;
    *d_desc = c->jobmem + (size_t)slot * SLOT_BYTES;
    *d_counter = reinterpret_cast<unsigned int*>(c->jobmem + JOB_SLOTS * SLOT_BYTES + (size_t)slot * 256);
    *d_tables = reinterpret_cast<uint32_t*>(c->jobmem + head);
    CK(cudaMemcpyAsync(*d_desc, desc, desc_bytes, cudaMemcpyHostToDevice, c->stream));
    CK(cudaMemsetAsync(*d_counter, 0, 4, c->stream));
    return 0;
}

int tecdsa_ctx::launch_exp(const ExpLaunch& l, int K) {
    JobGeom g = K == 32 ? job_geom<32, TPI_1024>(sm_count) : K == 64 ? job_geom<64, TPI_2048>(sm_count) : job_geom<128, TPI_4096>(sm_count);
    char* d_desc; unsigned int* d_counter; uint32_t* d_tables;
    int rc = job_prepare(this, g.table_bytes, &l, sizeof(ExpLaunch), &d_desc, &d_counter, &d_tables);
    if (rc) return rc;
    prof_begin(K == 32 ? "exp_jobs_kernel<32,4>" : K == 64 ? "exp_jobs_kernel<64,4>" : "exp_jobs_kernel<128,8>");
    if (K == 32) exp_jobs_kernel<32, TPI_1024><<<g.grid, JOB_BLOCK, 0, stream>>>(reinterpret_cast<const ExpLaunch*>(d_desc), d_tables, d_counter, d_work);
    else if (K == 64) exp_jobs_kernel<64, TPI_2048><<<g.grid, JOB_BLOCK, 0, stream>>>(reinterpret_cast<const ExpLaunch*>(d_desc), d_tables, d_counter, d_work);
    else exp_jobs_kernel<128, TPI_4096><<<g.grid, JOB_BLOCK, 0, stream>>>(reinterpret_cast<const ExpLaunch*>(d_desc), d_tables, d_counter, d_work);
    prof_end();
    count_launch();
    CK(cudaGetLastError());
    return 0;
}
namespace {
// defaults measured on an H100 at 400 W, 8192-session batch: 4 blocks of 128 threads per SM (128 registers, no spills, 16 warps);
// one block per SM makes the N-adic kernel 4 % slower, 4 lanes x 3 blocks 3 %; the p-adic alternatives are no faster
struct NadicShape { int tpi = 8, minb = 4, tpi32 = 4, minb32 = 4; };
// TECDSA_NADIC_SHAPE="<tpi>,<minb>[,<tpi32>,<minb32>]": lanes per group and min blocks per SM of the N-adic kernels (K = 64 and K = 32)
const NadicShape& nadic_shape() {
    static const NadicShape sh = [] {
        NadicShape s;
        if (const char* e = getenv("TECDSA_NADIC_SHAPE")) {
            int t = 0, b = 0, t2 = 0, b2 = 0;
            const int n = sscanf(e, "%d,%d,%d,%d", &t, &b, &t2, &b2);
            if (n >= 2 && ((t == 4 && (b == 1 || b == 3)) || (t == 8 && (b == 1 || b == 4)))) { s.tpi = t; s.minb = b; }
            if (n == 4 && ((t2 == 4 && (b2 == 1 || b2 == 4)) || (t2 == 2 && b2 == 1))) { s.tpi32 = t2; s.minb32 = b2; }
        }
        return s;
    }();
    return sh;
}
template <int K, int TPI, int MINB>
int launch_nadic_shape(tecdsa_ctx* c, const ExpLaunch& l) {
    int per_sm = 0;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, nadic_jobs_kernel<K, TPI, MINB>, JOB_BLOCK, 0);
    if (per_sm < 1) per_sm = 1;
    const int grid = c->sm_count * per_sm;
    const size_t table_bytes = (size_t)grid * (JOB_BLOCK / 32) * (32 / TPI) * (size_t)NADIC_TABLE_ENTRIES * 2 * K * 4;
    char* d_desc; unsigned int* d_counter; uint32_t* d_tables;
    int rc = job_prepare(c, table_bytes, &l, sizeof(ExpLaunch), &d_desc, &d_counter, &d_tables);
    if (rc) return rc;
    // the profile keeps the pointer: one static label per instantiation, naming all three parameters so every shape is told apart
    static const struct Label { char s[48]; Label() { snprintf(s, sizeof(s), "nadic_jobs_kernel<%d,%d,%d>", K, TPI, MINB); } } label;
    c->prof_begin(label.s);
    nadic_jobs_kernel<K, TPI, MINB><<<grid, JOB_BLOCK, 0, c->stream>>>(reinterpret_cast<const ExpLaunch*>(d_desc), d_tables, d_counter, c->d_work);
    c->prof_end();
    c->count_launch();
    CK(cudaGetLastError());
    return 0;
}
}  // namespace
namespace tecdsa {
int tecdsa_nadic_tpi() { return nadic_shape().tpi; }
int tecdsa_nadic32_tpi() { return nadic_shape().tpi32; }
bool tecdsa_hensel_inverse() {
    static const bool on = [] { const char* e = getenv("TECDSA_HENSEL"); return !(e && atoi(e) == 0); }();
    return on;
}
int tecdsa_nadic_minb() { return nadic_shape().minb; }
}

int tecdsa_ctx::launch_nadic(const ExpLaunch& l, int K) {
    for (int i = 0; i < l.n_classes; i++)
        if (!l.cls[i].nadic.ptr || l.cls[i].fb) return tecdsa_fail(TECDSA_E_ARG, "launch_nadic: class without N-adic constants");
    const NadicShape& sh = nadic_shape();
    if (K == 32) {
        if (sh.tpi32 == 2) return launch_nadic_shape<32, 2, 1>(this, l);
        return sh.minb32 == 4 ? launch_nadic_shape<32, 4, 4>(this, l) : launch_nadic_shape<32, 4, 1>(this, l);
    }
    if (sh.tpi == 8) return sh.minb == 4 ? launch_nadic_shape<64, 8, 4>(this, l) : launch_nadic_shape<64, 8, 1>(this, l);
    return sh.minb == 3 ? launch_nadic_shape<64, 4, 3>(this, l) : launch_nadic_shape<64, 4, 1>(this, l);
}
int tecdsa_ctx::launch_nadic_inv(const InvLaunch& l) {
    for (int i = 0; i < l.n_classes; i++)
        if (!l.cls[i].nadic.ptr) return tecdsa_fail(TECDSA_E_ARG, "launch_nadic_inv: class without N-adic constants");
    char* d_desc; unsigned int* d_counter; uint32_t* d_tables;
    int rc = job_prepare(this, 0, &l, sizeof(InvLaunch), &d_desc, &d_counter, &d_tables);
    if (rc) return rc;
    int per_sm = 0;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, nadic_inv_kernel<64, TPI_NADIC_INV>, JOB_BLOCK, 0);
    if (per_sm < 1) per_sm = 1;
    prof_begin("nadic_inv_kernel<64,8>");
    nadic_inv_kernel<64, TPI_NADIC_INV><<<sm_count * per_sm, JOB_BLOCK, 0, stream>>>(reinterpret_cast<const InvLaunch*>(d_desc), d_counter);
    prof_end();
    count_launch();
    CK(cudaGetLastError());
    return 0;
}
int tecdsa_ctx::nadic_setup(const uint32_t* n_tab, uint32_t* out, int rows, int K) {
    if (rows <= 0) return 0;
    const int per_block = JOB_BLOCK / 8;
    if (K == 32) nadic_setup_kernel<32, 8><<<(rows + per_block - 1) / per_block, JOB_BLOCK, 0, stream>>>(n_tab, out, rows);
    else nadic_setup_kernel<64, 8><<<(rows + per_block - 1) / per_block, JOB_BLOCK, 0, stream>>>(n_tab, out, rows);
    count_launch();
    CK(cudaGetLastError());
    return 0;
}
int tecdsa_ctx::launch_inv(const InvLaunch& l, int K) {
    char* d_desc; unsigned int* d_counter; uint32_t* d_tables;
    int rc = job_prepare(this, 0, &l, sizeof(InvLaunch), &d_desc, &d_counter, &d_tables);
    if (rc) return rc;
    int per_sm = 0;
    if (K == 64) cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, inv_jobs_kernel<64, TPI_2048>, JOB_BLOCK, 0);
    else cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, inv_jobs_kernel<128, TPI_4096>, JOB_BLOCK, 0);
    if (per_sm < 1) per_sm = 1;
    const int grid = sm_count * per_sm;
    prof_begin(K == 64 ? "inv_jobs_kernel<64,4>" : "inv_jobs_kernel<128,8>");
    if (K == 64) inv_jobs_kernel<64, TPI_2048><<<grid, JOB_BLOCK, 0, stream>>>(reinterpret_cast<const InvLaunch*>(d_desc), d_counter);
    else inv_jobs_kernel<128, TPI_4096><<<grid, JOB_BLOCK, 0, stream>>>(reinterpret_cast<const InvLaunch*>(d_desc), d_counter);
    prof_end();
    count_launch();
    CK(cudaGetLastError());
    return 0;
}
