// Engine context shared by the translation units of the library (see include/tecdsa_b200.h).
#pragma once
#include "../../include/tecdsa_b200.h"
#include "gg20_fields.h"

#include <cuda_runtime.h>
#include <cstdint>
#include <cstring>
#include <vector>

namespace tecdsa {
struct ExpLaunch;
struct InvLaunch;
// lane-group widths of the job-list kernels working directly on a K-limb modulus
constexpr int TPI_1024 = 4;     // 8 limbs per lane
constexpr int TPI_2048 = 4;     // 16 limbs per lane
constexpr int TPI_4096 = 8;     // 16 limbs per lane (generic 4096-bit moduli of the L0 entry points; the gg20 driver has none left)
// Jobs modulo a square (N^2 with 64-limb N; p^2, q^2 with 32-limb primes) run in N-adic form (nadic.cuh): lane groups are as
// wide as the ROOT.  The kernel shapes (lanes per group, min blocks per SM) are process-wide tuning choices:
// TECDSA_NADIC_SHAPE="<tpi>,<minb>[,<tpi32>,<minb32>]" overrides the defaults for measurements.
constexpr int NADIC_ROW = 10;       // constants row of a modulus: 10 * K limbs (nadic.cuh)
constexpr int TPI_NADIC_INV = 8;    // nadic_inv_kernel<64, .>
int tecdsa_nadic_tpi();             // K = 64
int tecdsa_nadic32_tpi();           // K = 32
int tecdsa_nadic_minb();
bool tecdsa_hensel_inverse();       // inverses modulo N^2 through nadic_inv_kernel; TECDSA_HENSEL=0 selects the 4096-bit Kaliski inversion
}  // namespace tecdsa

int tecdsa_fail(int code, const char* what, cudaError_t e = cudaSuccess);
// per-device fixed-base point tables (G, base_point2): built once, shared by every context of the device
int tecdsa_internal_fb_points_init(int device, cudaStream_t stream, const uint32_t** table_out);   // gg20.cu
int tecdsa_internal_fb_points_set_l12(const uint32_t* table);                                        // l12.cu
int tecdsa_internal_fb_points_set_keygen(const uint32_t* table);                                     // keygen.cu
int tecdsa_internal_fb_points_set_records(const uint32_t* table);                                    // records.cu
int tecdsa_internal_fb_points_set_ecops(const uint32_t* table);                                      // ecops.cu
int tecdsa_internal_fb_points_set_blame(const uint32_t* table);                                      // blame.cu
int tecdsa_internal_fb_points_set_lindell17(const uint32_t* table);                                  // lindell17.cu
int tecdsa_internal_fb_points_set_gg18(const uint32_t* table);                                       // gg18.cu

// the offline stage with a HOST copy of the session descriptors; rnd / outputs live where `mem` says (gg20.cu)
int tecdsa_internal_offline(tecdsa_ctx* c, const tecdsa_keyset* ks, const uint32_t* h_sessions, size_t n_sessions, const uint32_t* rnd,
                            uint8_t* status, uint32_t* R_out, uint32_t* sigma_out, uint32_t* tvec_out, uint32_t* digest_out, int mem);

#define CK(call)                                                               \
    do {                                                                       \
        cudaError_t _e = (call);                                               \
        if (_e != cudaSuccess) return tecdsa_fail(TECDSA_E_CUDA, #call, _e);   \
    } while (0)

struct tecdsa_keyset {
    uint32_t* mem = nullptr;
    uint32_t* tab[tecdsa::KT_COUNT] = {};
    uint32_t* ypk = nullptr;
    uint32_t* fb = nullptr;      // fixed-base tables of (h1, h2) per key row, see jobs.cuh
    uint32_t* nadic = nullptr;   // [rows][10*64] N-adic constants of the Paillier moduli N, see nadic.cuh
    uint32_t* nadic_p = nullptr; // [rows][10*32] the same for the primes p and q (jobs modulo p^2, q^2)
    uint32_t* nadic_q = nullptr;
    // sliding-window digits (recode.h) of the exponents N, p, q, p-1, q-1: rec[t] = [rows][32 * KEY_SIZE[t]] bytes inside
    // rec_mem, nullptr for the other tables
    uint8_t* rec_mem = nullptr;
    const uint8_t* rec[tecdsa::KT_COUNT] = {};
    int n_keysets = 0;
    int parties = 3;             // key rows per key set: row = keyset * parties + party (tecdsa_keys_upload_parties)
};

struct tecdsa_ctx {
    int device = 0;
    int sm_count = 0;
    cudaStream_t stream = nullptr;
    char* ws = nullptr;            // modexp_batch workspace (window tables + staging)
    size_t ws_bytes = 0;
    char* jobmem = nullptr;        // job-list launches: descriptor ring, counters, window tables
    size_t jobmem_bytes = 0;
    int job_slot = 0;
    char* rec = nullptr;           // staging of tecdsa_gg20_offline_records (inputs, per-unit outputs, packed records)
    size_t rec_bytes = 0;
    unsigned long long* d_work = nullptr;   // executed-work counter of the job kernels (MAC32), see tecdsa_ctx_work
    char* arena = nullptr;         // per-unit state of the last gg20 batch
    size_t arena_bytes = 0;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    float last_ms = 0.f;
    int last_launches = 0;
    uint64_t launches = 0;
    int tpi[3] = {0, 0, 0};        // modexp_batch override for 1024, 2048, 4096
    bool opt_sqr = false;          // modexp_batch: squarings through mont_sqr (sqr.cuh); see tecdsa_ctx_set_option
    int last_U = 0;
    // large gg20 batches run as two half-batches on two private streams (gg20.cu): the tail of one half's persistent
    // launch and its latency-bound glue kernels overlap the other half's job lists
    tecdsa_ctx* child[2] = {nullptr, nullptr};
    cudaEvent_t ev_fork = nullptr, ev_join[2] = {nullptr, nullptr};
    bool owns_stream = false;
    uint32_t last_off[tecdsa::F_COUNT] = {};

    // per-launch profiling (tecdsa_ctx_profile): CUDA events around every kernel launch of this context + a snapshot of the
    // executed-work counter after it; batches run unsplit (one stream) while it is on
    struct ProfEntry { const char* name; cudaEvent_t e0, e1; };
    bool profiling = false;
    std::vector<ProfEntry> prof;
    unsigned long long* prof_work = nullptr;      // pinned host: d_work after launch i
    size_t prof_cap = 0;
    unsigned long long prof_work_base = 0;
    void prof_begin(const char* name);
    void prof_end();

    void count_launch() { launches++; }
    int reserve_arena(size_t bytes);
    int launch_exp(const tecdsa::ExpLaunch& l, int K);
    int launch_inv(const tecdsa::InvLaunch& l, int K);
    int launch_nadic(const tecdsa::ExpLaunch& l, int K);                        // every class modulo a square (ExpClass::nadic set); K = limbs of the root
    int launch_nadic_inv(const tecdsa::InvLaunch& l);                           // inverses modulo N^2 (InvClass::nadic set), K = 64
    int nadic_setup(const uint32_t* n_tab, uint32_t* out, int rows, int K);    // device pointers; out = [rows][NADIC_ROW*K]
};
