// Result records of the batched offline stage, their single multi-GPU gather, and the online step.
//
//  * the 256-byte record per unit (SURVEY.md section 8e): status | R | sigma_i | k_i | t_vec | transcript digest — the
//    fields of `CompletedOfflineStage` (/root/reference/src/protocols/multi_party_ecdsa/gg_2020/state_machine/sign/
//    rounds.rs:647-654) in the reference's byte encodings (`Point::to_bytes(true)`, big-endian scalars);
//  * tecdsa_gather_results: ONE ncclAllGather of the per-rank record blocks over NVLink (units are independent, there is no
//    other exchange on the path).  NCCL is bound at run time (dlopen of the libnccl.so.2 already in the process, e.g. the
//    one torch loaded), so the library has no link-time dependency on it and single-GPU use never touches it;
//  * tecdsa_gg20_offline_records: host buffers in, host records out — H2D, seven rounds, pack, gather, D2H on the context
//    stream (the end-to-end call bench.py times);
//  * the online step `LocalSignature::{phase7_local_sig, output_signature}` + `verify`
//    (gg_2020/party_i.rs:850-936) for a batch of sessions.
#include "stage.cuh"

#include <dlfcn.h>
#include <string>
#include <mutex>

using namespace tecdsa;

int tecdsa_internal_fb_points_set_records(const uint32_t* table) {
    CK(cudaMemcpyToSymbol(secp::g_fb_points, &table, sizeof(table)));
    return 0;
}

namespace {

__device__ __forceinline__ void put_be32(uint8_t* out, const uint32_t* limbs8) {
    for (int i = 0; i < 32; i++) out[i] = (uint8_t)(limbs8[7 - (i >> 2)] >> (8 * (3 - (i & 3))));
}
__device__ __forceinline__ void put_point33(uint8_t* out, const uint32_t* xy16) {
    Affine a = affine_load(xy16);
    if (a.inf) { for (int i = 0; i < 33; i++) out[i] = 0; return; }
    affine_compress(out, a);
}
// one thread per unit
__global__ void k_pack_records(const uint8_t* status, const uint32_t* R, const uint32_t* sigma, const uint32_t* tvec, const uint32_t* digest,
                               const uint32_t* rnd, uint8_t* records, int units) {
    int u = blockIdx.x * blockDim.x + threadIdx.x;
    if (u >= units) return;
    uint8_t* r = records + (size_t)u * TECDSA_REC_BYTES;
    for (int i = 0; i < TECDSA_REC_BYTES; i += 4) *reinterpret_cast<uint32_t*>(r + i) = 0;
    r[TECDSA_REC_STATUS] = status[u];
    put_point33(r + TECDSA_REC_R, R + (size_t)u * 16);
    put_be32(r + TECDSA_REC_SIGMA, sigma + (size_t)u * 8);
    U256 k = load_scalar(rnd + (size_t)u * RND_LIMBS + RND_K);                  // SignKeys.k_i (party_i.rs:565), reduced like Scalar::from
    put_be32(r + TECDSA_REC_K, k.v);
    put_point33(r + TECDSA_REC_T0, tvec + (size_t)u * 32);
    put_point33(r + TECDSA_REC_T1, tvec + (size_t)u * 32 + 16);
    put_be32(r + TECDSA_REC_DIGEST, digest + (size_t)u * 8);
}

// LocalSignature::phase7_local_sig (party_i.rs:850-871): s_i = m * k_i + r * sigma_i with r = R.x mod q
__global__ void k_local_sig(const uint32_t* msg, const uint32_t* R, const uint32_t* sigma, const uint32_t* k, uint32_t* s_i, int units) {
    int u = blockIdx.x * blockDim.x + threadIdx.x;
    if (u >= units) return;
    const U256 m = sc_from_limbs(msg + (size_t)(u >> 1) * 8, 8);
    const U256 r = sc_reduce_once(u256_load(R + (size_t)u * 16), 0);
    u256_store(s_i + (size_t)u * 8, sc_add(sc_mul(m, load_scalar(k + (size_t)u * 8)), sc_mul(r, load_scalar(sigma + (size_t)u * 8))));
}
// LocalSignature::output_signature (party_i.rs:873-910) for two signers, then `verify` (party_i.rs:913-936): one thread per session
__global__ void k_output_signature(const uint32_t* msg, const uint32_t* R, const uint32_t* s_i, const uint32_t* y, const uint32_t* keyset,
                                   uint32_t* sig_r, uint32_t* sig_s, uint8_t* recid, uint8_t* status, int sessions) {
    int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= sessions) return;
    const Affine Rp = affine_load(R + (size_t)(2 * s) * 16);
    U256 sum = sc_add(load_scalar(s_i + (size_t)(2 * s) * 8), load_scalar(s_i + (size_t)(2 * s + 1) * 8));
    const U256 r = sc_reduce_once(Rp.x, 0);
    uint8_t rid = (uint8_t)(sc_reduce_once(Rp.y, 0).v[0] & 1u);          // `ry.mod_floor(q).test_bit(0)`
    U256 neg = sc_neg(sum);                                               // s > q - s  =>  s = q - s, recid ^= 1 (:896-902)
    bool flip = false;
    for (int i = 7; i >= 0; i--) { if (sum.v[i] != neg.v[i]) { flip = sum.v[i] > neg.v[i]; break; } }
    if (flip) { sum = neg; rid ^= 1; }
    u256_store(sig_r + (size_t)s * 8, r); u256_store(sig_s + (size_t)s * 8, sum);
    recid[s] = rid;
    // verify: b = s^-1, u1 = m b, u2 = r b, (u1 G + u2 y).x mod q == r
    bool ok = !Rp.inf && !u256_is_zero(sum) && !u256_is_zero(r);
    if (ok) {
        const U256 b = sc_inv(sum);
        const U256 u1 = sc_mul(sc_from_limbs(msg + (size_t)s * 8, 8), b), u2 = sc_mul(r, b);
        const Affine Y = affine_load(y + (size_t)keyset[s] * 16);
        const Affine P = lin_GP(u1, Y, u2);
        ok = !P.inf && u256_eq(sc_reduce_once(P.x, 0), r);
    }
    status[s] = ok ? TECDSA_ST_OK : TECDSA_ST_INVALID_SIG;
}

// ---- NCCL through dlopen ------------------------------------------------------------------------
struct NcclId { char internal[128]; };
struct NcclApi {
    void* so = nullptr;
    int (*GetUniqueId)(NcclId*) = nullptr;
    int (*CommInitRank)(void**, int, NcclId, int) = nullptr;
    int (*CommDestroy)(void*) = nullptr;
    int (*CommCount)(void*, int*) = nullptr;
    int (*AllGather)(const void*, void*, size_t, int, void*, cudaStream_t) = nullptr;
    const char* (*GetErrorString)(int) = nullptr;
};
NcclApi* nccl_api() {
    static NcclApi api;
    static std::once_flag once;
    std::call_once(once, [] {
        // prefer the copy already mapped into the process (torch brings its own libnccl.so.2); never load a second one
        void* so = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD | RTLD_GLOBAL);
        if (!so) so = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
        if (!so) so = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
        if (!so) return;
        api.so = so;
        api.GetUniqueId = reinterpret_cast<int (*)(NcclId*)>(dlsym(so, "ncclGetUniqueId"));
        api.CommInitRank = reinterpret_cast<int (*)(void**, int, NcclId, int)>(dlsym(so, "ncclCommInitRank"));
        api.CommDestroy = reinterpret_cast<int (*)(void*)>(dlsym(so, "ncclCommDestroy"));
        api.CommCount = reinterpret_cast<int (*)(void*, int*)>(dlsym(so, "ncclCommCount"));
        api.AllGather = reinterpret_cast<int (*)(const void*, void*, size_t, int, void*, cudaStream_t)>(dlsym(so, "ncclAllGather"));
        api.GetErrorString = reinterpret_cast<const char* (*)(int)>(dlsym(so, "ncclGetErrorString"));
    });
    if (!api.so || !api.GetUniqueId || !api.CommInitRank || !api.CommDestroy || !api.AllGather || !api.CommCount) return nullptr;
    return &api;
}
int nccl_fail(NcclApi* a, const char* what, int rc) {
    std::string m = what;
    if (a && a->GetErrorString) { m += ": "; m += a->GetErrorString(rc); }
    return tecdsa_fail(TECDSA_E_CUDA, m.c_str());
}
constexpr int NCCL_UINT8 = 1;      // ncclUint8 in nccl.h (ncclInt8 = 0, ncclUint8 = 1, ncclInt32 = 2, ...)

int grow_rec(tecdsa_ctx* c, size_t need) {
    if (need <= c->rec_bytes) return 0;
    CK(cudaStreamSynchronize(c->stream));
    if (c->rec) CK(cudaFree(c->rec));
    c->rec = nullptr; c->rec_bytes = 0;
    cudaError_t e = cudaMalloc(&c->rec, need);
    if (e != cudaSuccess) return tecdsa_fail(TECDSA_E_NOMEM, "cudaMalloc(record staging)", e);
    c->rec_bytes = need;
    return 0;
}
size_t al256(size_t x) { return (x + 255) & ~size_t(255); }

}  // namespace

extern "C" int tecdsa_nccl_unique_id(uint8_t id[TECDSA_NCCL_ID_BYTES]) {
    if (!id) return tecdsa_fail(TECDSA_E_ARG, "nccl_unique_id: null argument");
    NcclApi* a = nccl_api();
    if (!a) return tecdsa_fail(TECDSA_E_UNSUPPORTED, "NCCL (libnccl.so.2) is not available in this process");
    NcclId nid;
    int rc = a->GetUniqueId(&nid);
    if (rc) return nccl_fail(a, "ncclGetUniqueId", rc);
    memcpy(id, nid.internal, sizeof(nid.internal));
    return 0;
}
extern "C" int tecdsa_nccl_comm_create(tecdsa_ctx* c, const uint8_t id[TECDSA_NCCL_ID_BYTES], int nranks, int rank, void** comm) {
    if (!c || !id || !comm || nranks < 1 || rank < 0 || rank >= nranks) return tecdsa_fail(TECDSA_E_ARG, "nccl_comm_create: bad argument");
    NcclApi* a = nccl_api();
    if (!a) return tecdsa_fail(TECDSA_E_UNSUPPORTED, "NCCL (libnccl.so.2) is not available in this process");
    CK(cudaSetDevice(c->device));
    NcclId nid;
    memcpy(nid.internal, id, sizeof(nid.internal));
    int rc = a->CommInitRank(comm, nranks, nid, rank);
    if (rc) return nccl_fail(a, "ncclCommInitRank", rc);
    return 0;
}
extern "C" int tecdsa_nccl_comm_destroy(void* comm) {
    if (!comm) return 0;
    NcclApi* a = nccl_api();
    if (!a) return tecdsa_fail(TECDSA_E_UNSUPPORTED, "NCCL (libnccl.so.2) is not available in this process");
    int rc = a->CommDestroy(comm);
    return rc ? nccl_fail(a, "ncclCommDestroy", rc) : 0;
}

extern "C" int tecdsa_gg20_pack_records(tecdsa_ctx* c, const uint8_t* status, const uint32_t* R, const uint32_t* sigma, const uint32_t* t_vec,
                                        const uint32_t* digest, const uint32_t* rnd, size_t n_units, uint8_t* records) {
    if (!c || !status || !R || !sigma || !t_vec || !digest || !rnd || !records) return tecdsa_fail(TECDSA_E_ARG, "pack_records: null argument");
    if (n_units == 0) return 0;
    CK(cudaSetDevice(c->device));
    k_pack_records<<<grid_for(n_units), 64, 0, c->stream>>>(status, R, sigma, t_vec, digest, rnd, records, (int)n_units);
    c->count_launch();
    CK(cudaGetLastError());
    return 0;
}

extern "C" int tecdsa_gather_results(tecdsa_ctx* c, void* nccl_comm, const uint8_t* records, size_t n_units, uint8_t* all_records) {
    if (!c || !records || !all_records) return tecdsa_fail(TECDSA_E_ARG, "gather_results: null argument");
    CK(cudaSetDevice(c->device));
    const size_t bytes = n_units * TECDSA_REC_BYTES;
    if (!nccl_comm) {                                  // one rank: the gather is the identity
        if (all_records != records) CK(cudaMemcpyAsync(all_records, records, bytes, cudaMemcpyDeviceToDevice, c->stream));
        return 0;
    }
    NcclApi* a = nccl_api();
    if (!a) return tecdsa_fail(TECDSA_E_UNSUPPORTED, "NCCL (libnccl.so.2) is not available in this process");
    int rc = a->AllGather(records, all_records, bytes, NCCL_UINT8, nccl_comm, c->stream);
    return rc ? nccl_fail(a, "ncclAllGather", rc) : 0;
}

extern "C" int tecdsa_gg20_offline_records(tecdsa_ctx* c, const tecdsa_keyset* ks, void* nccl_comm, const uint32_t* sessions, size_t n_sessions,
                                           const uint32_t* rnd, uint8_t* all_records, int mem) {
    if (!c || !ks || !sessions || !rnd || !all_records) return tecdsa_fail(TECDSA_E_ARG, "gg20_offline_records: null argument");
    if (ks->parties != 3) return tecdsa_fail(TECDSA_E_ARG, "gg20_offline_records: the key set must have three parties");
    if (mem != TECDSA_HOST && mem != TECDSA_DEVICE) return tecdsa_fail(TECDSA_E_ARG, "gg20_offline_records: bad mem");
    if (n_sessions == 0) return 0;
    if (n_sessions > (1u << 22)) return tecdsa_fail(TECDSA_E_ARG, "gg20_offline_records: too many sessions");
    CK(cudaSetDevice(c->device));
    int nranks = 1;
    if (nccl_comm) {
        NcclApi* a = nccl_api();
        if (!a) return tecdsa_fail(TECDSA_E_UNSUPPORTED, "NCCL (libnccl.so.2) is not available in this process");
        int rc = a->CommCount(nccl_comm, &nranks);
        if (rc) return nccl_fail(a, "ncclCommCount", rc);
    }
    const size_t U = 2 * n_sessions, rec_bytes = U * TECDSA_REC_BYTES;
    // staging: [rnd (HOST only)] status R sigma tvec digest records [all records (HOST, or when gathering)]
    const size_t o_rnd = 0, o_status = o_rnd + (mem == TECDSA_HOST ? al256(U * RND_LIMBS * 4) : 0), o_R = o_status + al256(U), o_sigma = o_R + al256(U * 64),
                 o_tvec = o_sigma + al256(U * 32), o_digest = o_tvec + al256(U * 128), o_rec = o_digest + al256(U * 32),
                 o_all = o_rec + al256(rec_bytes), total = o_all + (mem == TECDSA_HOST ? al256(rec_bytes * (size_t)nranks) : 0);
    int rc = grow_rec(c, total);
    if (rc) return rc;
    std::vector<uint32_t> h_copy;
    const uint32_t* h_sess = sessions;
    const uint32_t* d_rnd = rnd;
    if (mem == TECDSA_HOST) {
        CK(cudaMemcpyAsync(c->rec + o_rnd, rnd, U * RND_LIMBS * 4, cudaMemcpyHostToDevice, c->stream));
        d_rnd = reinterpret_cast<const uint32_t*>(c->rec + o_rnd);
    } else {
        h_copy.resize(n_sessions * 3);
        CK(cudaMemcpyAsync(h_copy.data(), sessions, h_copy.size() * 4, cudaMemcpyDeviceToHost, c->stream));
        CK(cudaStreamSynchronize(c->stream));
        h_sess = h_copy.data();
    }
    uint8_t* d_status = reinterpret_cast<uint8_t*>(c->rec + o_status);
    uint32_t *d_R = reinterpret_cast<uint32_t*>(c->rec + o_R), *d_sigma = reinterpret_cast<uint32_t*>(c->rec + o_sigma),
             *d_tvec = reinterpret_cast<uint32_t*>(c->rec + o_tvec), *d_digest = reinterpret_cast<uint32_t*>(c->rec + o_digest);
    uint8_t* d_rec = reinterpret_cast<uint8_t*>(c->rec + o_rec);
    uint8_t* d_all = mem == TECDSA_HOST ? reinterpret_cast<uint8_t*>(c->rec + o_all) : all_records;
    rc = tecdsa_internal_offline(c, ks, h_sess, n_sessions, d_rnd, d_status, d_R, d_sigma, d_tvec, d_digest, TECDSA_DEVICE);
    if (rc) return rc;
    rc = tecdsa_gg20_pack_records(c, d_status, d_R, d_sigma, d_tvec, d_digest, d_rnd, U, d_rec);
    if (rc) return rc;
    rc = tecdsa_gather_results(c, nccl_comm, d_rec, U, d_all);
    if (rc) return rc;
    if (mem == TECDSA_HOST) {
        CK(cudaMemcpyAsync(all_records, d_all, rec_bytes * (size_t)nranks, cudaMemcpyDeviceToHost, c->stream));
        CK(cudaStreamSynchronize(c->stream));
    }
    return 0;
}

// ---- online step ---------------------------------------------------------------------------------
extern "C" int tecdsa_gg20_sign_batch(tecdsa_ctx* c, const tecdsa_keyset* ks, const uint32_t* sessions, size_t n_sessions, const uint32_t* message,
                                      const uint32_t* R, const uint32_t* sigma, const uint32_t* k, uint32_t* s_i, uint32_t* sig_r, uint32_t* sig_s,
                                      uint8_t* recid, uint8_t* status, int mem) {
    if (!c || !ks || !sessions || !message || !R || !sigma || !k || !sig_r || !sig_s || !recid || !status) return tecdsa_fail(TECDSA_E_ARG, "gg20_sign: null argument");
    if (ks->parties != 3) return tecdsa_fail(TECDSA_E_ARG, "gg20_sign: the key set must have three parties");
    STAGE_PROLOGUE("gg20_sign", n_sessions);
    const size_t U = 2 * n_sessions;
    const uint32_t *dsess = S.in(sessions, n_sessions * 3), *dm = S.in(message, n_sessions * 8), *dR = S.in(R, U * 16), *dsg = S.in(sigma, U * 8), *dk = S.in(k, U * 8);
    uint32_t* dsi = s_i ? S.out(s_i, U * 8) : S.tmp<uint32_t>(U * 8);
    uint32_t *dr = S.out(sig_r, n_sessions * 8), *ds = S.out(sig_s, n_sessions * 8);
    uint8_t *drec = S.out(recid, n_sessions), *dst = S.out(status, n_sessions);
    uint32_t* dkset = S.tmp<uint32_t>(n_sessions);
    if (S.err) return S.err;
    // the key set of a session is the first word of its descriptor
    if (cudaMemcpy2DAsync(dkset, 4, dsess, 12, 4, n_sessions, cudaMemcpyDeviceToDevice, c->stream) != cudaSuccess) return tecdsa_fail(TECDSA_E_CUDA, "gg20_sign: descriptor copy");
    k_local_sig<<<grid_for(U), 64, 0, c->stream>>>(dm, dR, dsg, dk, dsi, (int)U);
    KCHECK();
    k_output_signature<<<grid_for(n_sessions), 64, 0, c->stream>>>(dm, dR, dsi, ks->ypk, dkset, dr, ds, drec, dst, (int)n_sessions);
    KCHECK();
    return S.finish();
}

// ---- executed-work counter -----------------------------------------------------------------------
extern "C" int tecdsa_ctx_work(tecdsa_ctx* c, uint64_t* mac32, int reset) {
    if (!c) return tecdsa_fail(TECDSA_E_ARG, "ctx_work: null ctx");
    CK(cudaSetDevice(c->device));
    uint64_t total = 0;
    tecdsa_ctx* all[3] = {c, c->child[0], c->child[1]};
    for (tecdsa_ctx* x : all) {
        if (!x || !x->d_work) continue;
        unsigned long long v = 0;
        CK(cudaMemcpyAsync(&v, x->d_work, sizeof(v), cudaMemcpyDeviceToHost, x->stream));
        CK(cudaStreamSynchronize(x->stream));
        total += v;
        if (reset) CK(cudaMemsetAsync(x->d_work, 0, sizeof(v), x->stream));
    }
    if (mac32) *mac32 = total;
    return 0;
}
