// Key-generation path of GG20 (SURVEY.md section 8(f) rank 1), batched: the checks one party runs on every other party's
// KeyGenBroadcastMessage1 / Feldman shares and the proofs it produces itself
// (/root/reference/src/protocols/multi_party_ecdsa/gg_2020/party_i.rs:137-156,219-367,405-438).  Proof bodies are zk-paillier
// 0.4.3 / curv 0.9 (out of tree, [R]); oracle: oracle/keygen_oracle.py.
#include "stage.cuh"
#include "primorial.h"
#include "even_inverse.cuh"
#include "keygen_kernels.cuh"

using namespace tecdsa;

#include <climits>

int tecdsa_internal_fb_points_set_keygen(const uint32_t* table) {
    CK(cudaMemcpyToSymbol(secp::g_fb_points, &table, sizeof(table)));
    return 0;
}

// ------------------------------------------------------------------------------------------ key-generation verification path
namespace {

// out[i] = CONST mod n[i] for a public constant of `chunks` K-limb chunks (Horner over the chunks in the Montgomery domain of
// n[i]); one lane group per modulus.  Used for the primorial of NiCorrectKeyProof::verify: gcd(P, N) == gcd(P mod N, N).
// An even n has no Montgomery domain: its output is zero (callers reject even N separately — 2 divides the primorial).
template <int K, int TPI>
__global__ void __launch_bounds__(128)
const_mod_kernel(const uint32_t* __restrict__ n_tab, const uint32_t* __restrict__ cst, int chunks, uint32_t* __restrict__ out, int count) {
    constexpr int L = K / TPI;
    const int g = (blockIdx.x * blockDim.x + threadIdx.x) / TPI;
    const bool live = g < count;
    const int i = live ? g : count - 1;
    const int gl = group_lane<TPI>();
    MontCtx<L> m;
    load_limbs<TPI, L>(m.n, n_tab + (size_t)i * K);
    const bool odd = (__shfl_sync(FULL, m.n[0], 0, TPI) & 1u) != 0;
    if (gl == 0) m.n[0] |= 1u;
    mont_setup<TPI, L>(m);
    uint32_t acc[L], one_p[L], t[L];
#pragma unroll
    for (int j = 0; j < L; j++) { acc[j] = 0; one_p[j] = 0; }
    if (gl == 0) one_p[0] = 1;
#pragma unroll 1
    for (int h = chunks - 1; h >= 0; h--) {
        mont_mul<TPI, L>(acc, acc, m.rr, m.n, m.n0inv);                // acc * R mod n
        load_limbs<TPI, L>(t, cst + (size_t)h * K);
        mont_mul<TPI, L>(t, t, m.rr, m.n, m.n0inv);                    // chunk * R mod n (chunk < R, rr < n)
        mont_mul<TPI, L>(t, t, one_p, m.n, m.n0inv);                   // chunk mod n
        const uint32_t cy = group_add_masked<TPI, L>(acc, t, 0xffffffffu);
        uint32_t D[L];
#pragma unroll
        for (int j = 0; j < L; j++) D[j] = acc[j];
        const uint32_t ge = group_sub_masked<TPI, L>(D, m.n, 0xffffffffu, 1u);
        if (cy | ge) {
#pragma unroll
            for (int j = 0; j < L; j++) acc[j] = D[j];
        }
    }
    if (!odd) {
#pragma unroll
        for (int j = 0; j < L; j++) acc[j] = 0;
    }
    if (live) store_limbs<TPI, L>(out + (size_t)i * K, acc);
}

// instance t of a flat (key, j) batch belongs to key t / per
__global__ void k_iota_div(uint32_t* idx, int per, int total) {
    int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t < total) idx[t] = (uint32_t)(t / per);
}
// NiCorrectKeyProof::verify prologue (zk-paillier 0.4.3 correct_key_ni.rs [R]; call site gg_2020/party_i.rs:288-291):
// rho_j = mask_generation(|N|, H(N, salt, j)) for j < 11, left un-reduced (<= 72 limbs)
__global__ void k_ck_rho(const uint32_t* n_tab, const uint8_t* salt, int salt_len, uint32_t* rho72, int count) {
    int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= count * 11) return;
    const int i = t / 11, j = t % 11;
    const uint32_t* N = n_tab + (size_t)i * 64;
    int top = 63;
    while (top > 0 && N[top] == 0) top--;
    const int key_len = N[top] ? top * 32 + (32 - __clz(N[top])) : 0;
    Sha256 h; h.init();
    h.put_bigint(N, 64);
    {   // BigInt::from_bytes(salt).to_bytes(): leading zero bytes dropped, zero -> one 0x00
        int s0 = 0;
        while (s0 < salt_len - 1 && salt[s0] == 0) s0++;
        if (salt_len <= 0) h.put(0);
        else h.put_bytes(salt + s0, salt_len - s0);
    }
    uint32_t jj = (uint32_t)j;
    h.put_bigint(&jj, 1);
    uint32_t seed[8];
    h.finish(seed);
    uint32_t* out = rho72 + (size_t)t * 72;
    for (int k = 0; k < 72; k++) out[k] = 0;
    int msklen = key_len / 256 + 1;
    if (msklen > 9) msklen = 9;
    for (int m = 0; m < msklen; m++) {         // digests occupy disjoint 256-bit slots: the sum is a concatenation
        Sha256 g; g.init();
        g.put_bigint(seed, 8);
        uint32_t mm = (uint32_t)m;
        g.put_bigint(&mm, 1);
        g.finish(out + 8 * m);
    }
}
// accept iff gcd(P, N) == 1 (N odd and P mod N invertible modulo N) and sigma_j^N == rho_j for all j
__global__ void k_ck_cmp(const uint32_t* n_tab, const uint32_t* got, const uint32_t* want, const uint8_t* gcd_ok, uint8_t* status, int count) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    bool ok = gcd_ok[i] != 0 && (n_tab[(size_t)i * 64] & 1u);
    for (int j = 0; j < 11 && ok; j++) ok = st::cmp(got + ((size_t)i * 11 + j) * 64, want + ((size_t)i * 11 + j) * 64, 64) == 0;
    status[i] = ok ? TECDSA_ST_OK : TECDSA_ST_PROOF;
}
// CompositeDLogProof::verify prologue (zk-paillier 0.4.3 composite_dlog_proof.rs [R]; call sites party_i.rs:296-303):
// e = H(x, g, N, ni) and the N > 2^128 / odd-N preconditions
__global__ void k_cd_pre(const uint32_t* N, const uint32_t* g, const uint32_t* ni, const uint32_t* x, uint32_t* e8, uint8_t* pre_ok, int count) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    const uint32_t* n = N + (size_t)i * 64;
    Sha256 h; h.init();
    h.put_bigint(x + (size_t)i * 64, 64);
    h.put_bigint(g + (size_t)i * 64, 64);
    h.put_bigint(n, 64);
    h.put_bigint(ni + (size_t)i * 64, 64);
    h.finish(e8 + (size_t)i * 8);
    int top = 63;
    while (top > 0 && n[top] == 0) top--;
    bool big = top > 4 || (top == 4 && (n[4] > 1 || (n[0] | n[1] | n[2] | n[3]) != 0));
    pre_ok[i] = (big && (n[0] & 1u)) ? 1 : 0;
}
__global__ void k_cd_post(const uint32_t* v, const uint32_t* x, const uint8_t* pre_ok, const uint8_t* ok_g, const uint8_t* ok_ni, uint8_t* status, int count) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    const bool ok = pre_ok[i] && ok_g[i] && ok_ni[i] && st::cmp(v + (size_t)i * 64, x + (size_t)i * 64, 64) == 0;
    status[i] = ok ? TECDSA_ST_OK : TECDSA_ST_PROOF;
}
// curv VerifiableSS::validate_share [R] (call site party_i.rs:337-339): share * G == sum_j index^j * C_j (Horner)
__global__ void k_vss_validate(const uint32_t* commitments, int n_comm, const uint32_t* share, const uint32_t* index, uint8_t* status, int count) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    status[i] = kg::vss_share_ok(commitments + (size_t)i * n_comm * 16, n_comm, share + (size_t)i * 8, index[i]) ? TECDSA_ST_OK : TECDSA_ST_PROOF;
}


// NiCorrectKeyProof::verify on staged device buffers: n = [count][64], sigma = [count][11][64] -> status
int correct_key_verify_step(tecdsa_ctx* c, Stage& S, int n, const uint32_t* dn, const uint32_t* ds, const uint8_t* dsalt, int salt_len, uint8_t* dst) {
    const size_t count = (size_t)n;
    const int tot = n * 11;
    uint32_t *rho72 = S.tmp<uint32_t>((size_t)tot * 72), *rho = S.tmp<uint32_t>((size_t)tot * 64), *got = S.tmp<uint32_t>((size_t)tot * 64);
    uint32_t *idx = S.tmp<uint32_t>(tot), *one = S.tmp<uint32_t>(4), *pmod = S.tmp<uint32_t>(count * 64), *pinv = S.tmp<uint32_t>(count * 64);
    uint8_t* gcd_ok = S.tmp<uint8_t>(count);
    if (S.err) return S.err;
    static const uint32_t h_one[4] = {1, 0, 0, 0};
    if (cudaMemcpyAsync(one, h_one, sizeof(h_one), cudaMemcpyHostToDevice, c->stream) != cudaSuccess) return tecdsa_fail(TECDSA_E_CUDA, "correct_key_verify: H2D");
    k_iota_div<<<grid_for(tot), 64, 0, c->stream>>>(idx, 11, tot);
    KCHECK();
    k_ck_rho<<<grid_for(tot), 64, 0, c->stream>>>(dn, dsalt, salt_len, rho72, n);
    KCHECK();
    // gcd(P, N) == 1 for the primorial P of all primes <= 6379 [R]: P mod N, then the existence of its inverse modulo N
    {
        const uint32_t* prim = nullptr;
        if (cudaGetSymbolAddress((void**)&prim, PRIMORIAL_6379) != cudaSuccess) return tecdsa_fail(TECDSA_E_CUDA, "correct_key_verify: primorial symbol");
        const_mod_kernel<64, TPI_2048><<<(n + 128 / TPI_2048 - 1) / (128 / TPI_2048), 128, 0, c->stream>>>(dn, prim, PRIMORIAL_LIMBS / 64, pmod, n);
        KCHECK();
    }
    Launches L;
    add_inv(L.i64, 64, n, arr(dn, 64), arr(pmod, 64), pinv, gcd_ok);
    RUN(run(c, L.i64, 64));
    const Operand N = tab(dn, idx, 64);
    // rho mod N: the un-reduced mask as a double-width base to the power 1
    add_exp(L.e64, 64, tot, N, 1, arr(rho72, 72), Operand{one, nullptr, 0, 0, 4}, 1, NONE, NONE, 0, 0, NONE, NONE, rho, 64, 1);
    // sigma^N mod N (party_i.rs:288-291 -> correct_key_ni.rs verify [R])
    add_exp(L.e64, 64, tot, N, 1, arr(ds, 64), N, 64, NONE, NONE, 0, 0, NONE, NONE, got, 64);
    RUN(run(c, L.e64, 64));
    k_ck_cmp<<<grid_for(count), 64, 0, c->stream>>>(dn, got, rho, gcd_ok, dst, n);
    KCHECK();
    return 0;
}

// CompositeDLogProof::verify on staged device buffers
int composite_dlog_verify_step(tecdsa_ctx* c, Stage& S, int n, const uint32_t* dN, const uint32_t* dg, const uint32_t* dni, const uint32_t* dx,
                               const uint32_t* dy, int y_limbs, uint8_t* dst) {
    const size_t count = (size_t)n;
    uint32_t *e8 = S.tmp<uint32_t>(count * 8), *v = S.tmp<uint32_t>(count * 64), *scratch = S.tmp<uint32_t>(count * 64 * 2);
    uint8_t *pre_ok = S.tmp<uint8_t>(count), *ok_g = S.tmp<uint8_t>(count), *ok_ni = S.tmp<uint8_t>(count);
    if (S.err) return S.err;
    k_cd_pre<<<grid_for(count), 64, 0, c->stream>>>(dN, dg, dni, dx, e8, pre_ok, n);
    KCHECK();
    Launches L;
    // gcd(g, N) == 1 and gcd(ni, N) == 1 through the existence of the inverses
    add_inv(L.i64, 64, n, arr(dN, 64), arr(dg, 64), scratch, ok_g);
    add_inv(L.i64, 64, n, arr(dN, 64), arr(dni, 64), scratch + count * 64, ok_ni);
    RUN(run(c, L.i64, 64));
    // g^y * ni^e mod N (Straus double exponentiation)
    add_exp(L.e64, 64, n, arr(dN, 64), 2, arr(dg, 64), arr(dy, (uint32_t)y_limbs), y_limbs, arr(dni, 64), arr(e8, 8), 8, 0, NONE, NONE, v, 64);
    RUN(run(c, L.e64, 64));
    k_cd_post<<<grid_for(count), 64, 0, c->stream>>>(v, dx, pre_ok, ok_g, ok_ni, dst, n);
    KCHECK();
    return 0;
}

}  // namespace

extern "C" int tecdsa_correct_key_verify_batch(tecdsa_ctx* c, const uint32_t* n_mod, const uint32_t* sigma, const uint8_t* salt, int salt_len,
                                               uint8_t* status, size_t count, int mem) {
    if (!n_mod || !sigma || !status || salt_len < 0 || salt_len > 64 || (salt_len && !salt)) return tecdsa_fail(TECDSA_E_ARG, "correct_key_verify: bad argument");
    STAGE_PROLOGUE("correct_key_verify", count);
    const uint32_t *dn = S.in(n_mod, count * 64), *ds = S.in(sigma, count * 11 * 64);
    const uint8_t* dsalt = S.in(salt, (size_t)(salt_len ? salt_len : 0));
    uint8_t* dst = S.out(status, count);
    if (S.err) return S.err;
    RUN(correct_key_verify_step(c, S, (int)count, dn, ds, dsalt, salt_len, dst));
    return S.finish();
}

extern "C" int tecdsa_composite_dlog_verify_batch(tecdsa_ctx* c, const uint32_t* n_tilde, const uint32_t* g, const uint32_t* ni, const uint32_t* x,
                                                  const uint32_t* y, int y_limbs, uint8_t* status, size_t count, int mem) {
    if (!n_tilde || !g || !ni || !x || !y || !status || y_limbs <= 0 || y_limbs > 128) return tecdsa_fail(TECDSA_E_ARG, "composite_dlog_verify: bad argument");
    STAGE_PROLOGUE("composite_dlog_verify", count);
    const uint32_t *dN = S.in(n_tilde, count * 64), *dg = S.in(g, count * 64), *dni = S.in(ni, count * 64), *dx = S.in(x, count * 64);
    const uint32_t* dy = S.in(y, count * (size_t)y_limbs);
    uint8_t* dst = S.out(status, count);
    if (S.err) return S.err;
    RUN(composite_dlog_verify_step(c, S, (int)count, dN, dg, dni, dx, dy, y_limbs, dst));
    return S.finish();
}

extern "C" int tecdsa_vss_validate_share_batch(tecdsa_ctx* c, const uint32_t* commitments, int n_commitments, const uint32_t* share,
                                               const uint32_t* index, uint8_t* status, size_t count, int mem) {
    if (!commitments || !share || !index || !status || n_commitments <= 0 || n_commitments > 64) return tecdsa_fail(TECDSA_E_ARG, "vss_validate_share: bad argument");
    STAGE_PROLOGUE("vss_validate_share", count);
    const uint32_t *dc = S.in(commitments, count * (size_t)n_commitments * 16), *ds = S.in(share, count * 8), *di = S.in(index, count);
    uint8_t* dst = S.out(status, count);
    if (S.err) return S.err;
    k_vss_validate<<<grid_for(count), 64, 0, c->stream>>>(dc, n_commitments, ds, di, dst, (int)count);
    KCHECK();
    return S.finish();
}

// ------------------------------------------------------------------------------------------ key-generation PROVE side
// What one party computes for its own KeyGenBroadcastMessage1 / Feldman shares (party_i.rs:137-156, 219-258, 313): all
// randomness is an explicit input.  Inverses modulo the EVEN moduli phi(N) are obtained from an inversion modulo an odd number:
//     a^-1 mod m = (1 + m*t) / a,   t = -(m^-1) mod a          (a odd, gcd(a, m) = 1; the division is exact)
// so the Kaliski job list (odd moduli only) serves `BigInt::mod_inv(&xhi, &phi)` (party_i.rs:146) and N^-1 mod phi(N)
// (zk-paillier correct_key_ni.rs `proof` [R]).
namespace {

// zk-paillier `SALT_STRING` [R] ("KZen"): the salt of the NiCorrectKeyProof of key generation (party_i.rs:225,288-291)
const uint8_t KEYGEN_SALT[4] = {75, 90, 101, 110};
// CompositeDLogProof response width in key generation: y = r + e * (phi - xhi) < 2^512 + 2^2304 fits 73 limbs, rounded to 4
constexpr int CDL_Y_LIMBS = 76;

// CompositeDLogProof::prove tail (zk-paillier composite_dlog_proof.rs [R]; call sites party_i.rs:238-241):
// e = H(x, g, N, ni), y = r + e * secret over the integers
__global__ void k_cd_prove_post(const uint32_t* N, const uint32_t* g, const uint32_t* ni, const uint32_t* x, const uint32_t* secret, int secret_limbs,
                                const uint32_t* r16, uint32_t* y, int y_limbs, int count) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    uint32_t e[8];
    Sha256 h; h.init();
    h.put_bigint(x + (size_t)i * 64, 64);
    h.put_bigint(g + (size_t)i * 64, 64);
    h.put_bigint(N + (size_t)i * 64, 64);
    h.put_bigint(ni + (size_t)i * 64, 64);
    h.finish(e);
    st::mul_add(y + (size_t)i * y_limbs, y_limbs, e, 8, secret + (size_t)i * secret_limbs, secret_limbs, r16 + (size_t)i * 16, 16);
}
// VerifiableSS::share (curv [R]; call site party_i.rs:313): thread (i, j < t+1) the commitment a_j * G, thread (i, t+1+k) the
// share f(k+1) by Horner modulo q
__global__ void k_vss_share(const uint32_t* coeff, int t1, int n, uint32_t* shares, uint32_t* commitments, int count) {
    int id = blockIdx.x * blockDim.x + threadIdx.x;
    const int per = t1 + n;
    if (id >= count * per) return;
    const int i = id / per, j = id % per;
    const uint32_t* c = coeff + (size_t)i * t1 * 8;
    if (j < t1) {
        affine_store(commitments + ((size_t)i * t1 + j) * 16, mul_G(sc_from_limbs(c + (size_t)j * 8, 8)));
        return;
    }
    U256 xk = u256_zero(); xk.v[0] = (uint32_t)(j - t1 + 1);
    U256 acc = sc_from_limbs(c + (size_t)(t1 - 1) * 8, 8);
    for (int d = t1 - 2; d >= 0; d--) acc = sc_add(sc_mul(acc, xk), sc_from_limbs(c + (size_t)d * 8, 8));
    u256_store(shares + ((size_t)i * n + (j - t1)) * 8, acc);
}
__global__ void k_lin_sub(const uint32_t* a64, const uint32_t* b64, uint32_t* out64, int count) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < count) st::sub(out64 + (size_t)i * 64, a64 + (size_t)i * 64, b64 + (size_t)i * 64, 64);
}
__global__ void k_fill_u8(uint8_t* p, uint8_t v, int count) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < count) p[i] = v;
}

// NiCorrectKeyProof::proof(&dk, None) on staged device buffers; N = p*q is written to `N` [count][64]
int correct_key_prove_step(tecdsa_ctx* c, Stage& S, int n, const uint32_t* dp, const uint32_t* dq, const uint8_t* dsalt, int salt_len, uint32_t* dsig,
                           uint8_t* dst, uint32_t* N) {
    const size_t count = (size_t)n;
    const int tot = n * 11;
    uint32_t *phi = S.tmp<uint32_t>(count * 64), *phinv = S.tmp<uint32_t>(count * 64), *d = S.tmp<uint32_t>(count * 64);
    uint32_t *rho72 = S.tmp<uint32_t>((size_t)tot * 72), *rho = S.tmp<uint32_t>((size_t)tot * 64), *idx = S.tmp<uint32_t>(tot), *one = S.tmp<uint32_t>(4);
    uint8_t* ok = S.tmp<uint8_t>(count);
    if (S.err) return S.err;
    static const uint32_t h_one[4] = {1, 0, 0, 0};
    if (cudaMemcpyAsync(one, h_one, sizeof(h_one), cudaMemcpyHostToDevice, c->stream) != cudaSuccess) return tecdsa_fail(TECDSA_E_CUDA, "correct_key_prove: H2D");
    k_fill_u8<<<grid_for(count), 64, 0, c->stream>>>(dst, 0, n);
    KCHECK();
    k_kp_pre<<<grid_for(count), 64, 0, c->stream>>>(dp, dq, N, phi, n);
    KCHECK();
    k_iota_div<<<grid_for(tot), 64, 0, c->stream>>>(idx, 11, tot);
    KCHECK();
    k_ck_rho<<<grid_for(tot), 64, 0, c->stream>>>(N, dsalt, salt_len, rho72, n);
    KCHECK();
    Launches L;
    add_inv(L.i64, 64, n, arr(N, 64), arr(phi, 64), phinv, ok);                 // phi^-1 mod N (N odd)
    RUN(run(c, L.i64, 64));
    k_inv_even_post<<<grid_for(count), 64, 0, c->stream>>>(N, phi, phinv, ok, d, 0, dst, n);       // d = N^-1 mod phi
    KCHECK();
    const Operand Nt = tab(N, idx, 64);
    add_exp(L.e64, 64, tot, Nt, 1, arr(rho72, 72), Operand{one, nullptr, 0, 0, 4}, 1, NONE, NONE, 0, 0, NONE, NONE, rho, 64, 1);
    RUN(run(c, L.e64, 64));
    add_exp(L.e64, 64, tot, Nt, 1, arr(rho, 64), tab(d, idx, 64), 64, NONE, NONE, 0, 0, NONE, NONE, dsig, 64);
    RUN(run(c, L.e64, 64));
    return 0;
}

// CompositeDLogProof::prove on staged device buffers
int composite_dlog_prove_step(tecdsa_ctx* c, int n, const uint32_t* dN, const uint32_t* dg, const uint32_t* dni, const uint32_t* dsec, int secret_limbs,
                              const uint32_t* dr, uint32_t* dx, uint32_t* dy, int y_limbs) {
    Launches L;
    add_exp(L.e64, 64, n, arr(dN, 64), 1, arr(dg, 64), arr(dr, 16), 16, NONE, NONE, 0, 0, NONE, NONE, dx, 64);
    RUN(run(c, L.e64, 64));
    k_cd_prove_post<<<grid_for((size_t)n), 64, 0, c->stream>>>(dN, dg, dni, dx, dsec, secret_limbs, dr, dy, y_limbs, n);
    KCHECK();
    return 0;
}

// VerifiableSS::share on staged device buffers
int vss_share_step(tecdsa_ctx* c, int n, int t1, int n_shares, const uint32_t* dc, uint32_t* dsh, uint32_t* dcm) {
    k_vss_share<<<grid_for((size_t)n * (size_t)(t1 + n_shares)), 64, 0, c->stream>>>(dc, t1, n_shares, dsh, dcm, n);
    KCHECK();
    return 0;
}

// generate_h1_h2_N_tilde on staged device buffers
int h1_h2_n_tilde_step(tecdsa_ctx* c, Stage& S, int n, const uint32_t* dp, const uint32_t* dq, const uint32_t* dh1, const uint32_t* dxhi, uint32_t* dN,
                       uint32_t* dh2, uint32_t* dxn, uint32_t* dxin, uint8_t* dst) {
    const size_t count = (size_t)n;
    uint32_t *phi = S.tmp<uint32_t>(count * 64), *minv = S.tmp<uint32_t>(count * 64);
    uint8_t* ok = S.tmp<uint8_t>(count);
    if (S.err) return S.err;
    k_fill_u8<<<grid_for(count), 64, 0, c->stream>>>(dst, 0, n);
    KCHECK();
    k_kp_pre<<<grid_for(count), 64, 0, c->stream>>>(dp, dq, dN, phi, n);
    KCHECK();
    Launches L;
    add_exp(L.e64, 64, n, arr(dN, 64), 1, arr(dh1, 64), arr(dxhi, 64), 64, NONE, NONE, 0, 0, NONE, NONE, dh2, 64);
    RUN(run(c, L.e64, 64));
    add_inv(L.i64, 64, n, arr(dxhi, 64), arr(phi, 64), minv, ok);              // (phi mod xhi)^-1 mod xhi; an even xhi is caught below
    RUN(run(c, L.i64, 64));
    k_inv_even_post<<<grid_for(count), 64, 0, c->stream>>>(dxhi, phi, minv, ok, dxin, 1, dst, n);   // phi - xhi^-1 mod phi
    KCHECK();
    k_lin_sub<<<grid_for(count), 64, 0, c->stream>>>(phi, dxhi, dxn, n);
    KCHECK();
    return 0;
}

}  // namespace

// NiCorrectKeyProof::proof(&dk, None) (zk-paillier correct_key_ni.rs [R]; call site party_i.rs:225):
// sigma_j = rho_j^(N^-1 mod phi(N)) mod N for j < 11.  p, q = [count][32]; sigma = [count][11][64].
extern "C" int tecdsa_correct_key_prove_batch(tecdsa_ctx* c, const uint32_t* p, const uint32_t* q, const uint8_t* salt, int salt_len,
                                              uint32_t* sigma, uint8_t* status, size_t count, int mem) {
    if (!p || !q || !sigma || !status || salt_len < 0 || salt_len > 64 || (salt_len && !salt)) return tecdsa_fail(TECDSA_E_ARG, "correct_key_prove: bad argument");
    STAGE_PROLOGUE("correct_key_prove", count);
    const uint32_t *dp = S.in(p, count * 32), *dq = S.in(q, count * 32);
    const uint8_t* dsalt = S.in(salt, (size_t)(salt_len ? salt_len : 0));
    uint32_t* dsig = S.out(sigma, count * 11 * 64);
    uint8_t* dst = S.out(status, count);
    uint32_t* N = S.tmp<uint32_t>(count * 64);
    if (S.err) return S.err;
    RUN(correct_key_prove_step(c, S, (int)count, dp, dq, dsalt, salt_len, dsig, dst, N));
    return S.finish();
}

// CompositeDLogProof::prove(&DLogStatement{N, g, ni}, &secret) (party_i.rs:238-241): nonce r = [count][16] (< 2^512),
// secret = [count][secret_limbs]; x = g^r mod N [count][64], y = r + e*secret [count][y_limbs], y_limbs >= secret_limbs + 9.
extern "C" int tecdsa_composite_dlog_prove_batch(tecdsa_ctx* c, const uint32_t* n_tilde, const uint32_t* g, const uint32_t* ni, const uint32_t* secret,
                                                 int secret_limbs, const uint32_t* r, uint32_t* x, uint32_t* y, int y_limbs, size_t count, int mem) {
    if (!n_tilde || !g || !ni || !secret || !r || !x || !y || secret_limbs <= 0 || secret_limbs > 64 || y_limbs < secret_limbs + 9 || y_limbs > 128 || (y_limbs & 3))
        return tecdsa_fail(TECDSA_E_ARG, "composite_dlog_prove: bad argument");
    STAGE_PROLOGUE("composite_dlog_prove", count);
    const uint32_t *dN = S.in(n_tilde, count * 64), *dg = S.in(g, count * 64), *dni = S.in(ni, count * 64);
    const uint32_t *dsec = S.in(secret, count * (size_t)secret_limbs), *dr = S.in(r, count * 16);
    uint32_t *dx = S.out(x, count * 64), *dy = S.out(y, count * (size_t)y_limbs);
    if (S.err) return S.err;
    RUN(composite_dlog_prove_step(c, (int)count, dN, dg, dni, dsec, secret_limbs, dr, dx, dy, y_limbs));
    return S.finish();
}

// VerifiableSS::share(t, n, &secret) with explicit coefficients (party_i.rs:313): coefficients = [count][t+1][8] (index 0 = the
// secret) -> shares [count][n][8] = f(1..n) mod q, commitments [count][t+1][16] = a_j * G.
extern "C" int tecdsa_vss_share_batch(tecdsa_ctx* c, int t, int n_shares, const uint32_t* coefficients, uint32_t* shares, uint32_t* commitments,
                                      size_t count, int mem) {
    if (!coefficients || !shares || !commitments || t < 0 || t > 63 || n_shares <= 0 || n_shares > 4096) return tecdsa_fail(TECDSA_E_ARG, "vss_share: bad argument");
    STAGE_PROLOGUE("vss_share", count);
    const int t1 = t + 1;
    const uint32_t* dc = S.in(coefficients, count * (size_t)t1 * 8);
    uint32_t *dsh = S.out(shares, count * (size_t)n_shares * 8), *dcm = S.out(commitments, count * (size_t)t1 * 16);
    if (S.err) return S.err;
    RUN(vss_share_step(c, (int)count, t1, n_shares, dc, dsh, dcm));
    return S.finish();
}

// generate_h1_h2_N_tilde (party_i.rs:137-156) with its samples explicit: p~, q~ = [count][32] primes, h1 < N~, xhi < phi ->
// N~ = p~ q~, h2 = h1^xhi mod N~, and the NEGATED exponents phi - xhi, phi - xhi^-1 the function returns.  status NOT_INVERTIBLE
// where the reference's sampling loop would draw again (`mod_inv(&xhi, &phi)` is None, :146-149).
extern "C" int tecdsa_h1_h2_n_tilde_batch(tecdsa_ctx* c, const uint32_t* p_t, const uint32_t* q_t, const uint32_t* h1, const uint32_t* xhi,
                                          uint32_t* n_tilde, uint32_t* h2, uint32_t* xhi_neg, uint32_t* xhi_inv_neg, uint8_t* status, size_t count, int mem) {
    if (!p_t || !q_t || !h1 || !xhi || !n_tilde || !h2 || !xhi_neg || !xhi_inv_neg || !status) return tecdsa_fail(TECDSA_E_ARG, "h1_h2_n_tilde: bad argument");
    STAGE_PROLOGUE("h1_h2_n_tilde", count);
    const uint32_t *dp = S.in(p_t, count * 32), *dq = S.in(q_t, count * 32), *dh1 = S.in(h1, count * 64), *dxhi = S.in(xhi, count * 64);
    uint32_t *dN = S.out(n_tilde, count * 64), *dh2 = S.out(h2, count * 64), *dxn = S.out(xhi_neg, count * 64), *dxin = S.out(xhi_inv_neg, count * 64);
    uint8_t* dst = S.out(status, count);
    if (S.err) return S.err;
    RUN(h1_h2_n_tilde_step(c, S, (int)count, dp, dq, dh1, dxhi, dN, dh2, dxn, dxin, dst));
    return S.finish();
}

// ------------------------------------------------------------------------------------------ GG20 key generation, Round0..Round4
// (state_machine/keygen/rounds.rs:26-300) for `groups` groups of n parties in one staged call; see the header for the layouts.
// Every broadcast and every DLog proof is verified once per sender (every receiver runs the same deterministic check on the same
// message); the n^2 share validations run per (receiver, sender) pair.  All intermediates live in stage scratch.
extern "C" int tecdsa_gg20_keygen_batch(tecdsa_ctx* c, int t, int n, size_t groups, int mem, const tecdsa_keygen_in* in, const tecdsa_keygen_out* out) {
    if (t < 1 || t > n - 1 || n < 2 || n > 64 || !in || !out || groups > (size_t)(INT_MAX / 64) / (11 * (size_t)n))
        return tecdsa_fail(TECDSA_E_ARG, "gg20_keygen: bad argument");
    if (!in->paillier_p || !in->paillier_q || !in->n_tilde_p || !in->n_tilde_q || !in->u || !in->coeffs || !in->blind || !in->h1 || !in->xhi ||
        !in->cdl_nonce || !in->dlog_nonce || !out->x_i || !out->vss || !out->n || !out->dlog_st || !out->y || !out->pk || !out->status ||
        !out->bad_actors || !out->complete)
        return tecdsa_fail(TECDSA_E_ARG, "gg20_keygen: null buffer");
    const size_t E = groups * (size_t)n;
    STAGE_PROLOGUE("gg20_keygen", E);
    const int e = (int)E, t1 = t + 1;
    const size_t R = 64 * sizeof(uint32_t);                 // bytes of one 2048-bit row
    const uint32_t *dp = S.in(in->paillier_p, E * 32), *dq = S.in(in->paillier_q, E * 32), *dpt = S.in(in->n_tilde_p, E * 32), *dqt = S.in(in->n_tilde_q, E * 32);
    const uint32_t *du = S.in(in->u, E * 8), *da = S.in(in->coeffs, E * (size_t)t * 8), *dblind = S.in(in->blind, E * 8);
    const uint32_t *dh1 = S.in(in->h1, E * 64), *dxhi = S.in(in->xhi, E * 64), *dcdl = S.in(in->cdl_nonce, E * 32), *ddl = S.in(in->dlog_nonce, E * 8);
    uint32_t *ox = S.out(out->x_i, E * 8), *ovss = S.out(out->vss, E * (size_t)t1 * 16), *oN = S.out(out->n, E * 64), *ost = S.out(out->dlog_st, E * 3 * 64);
    uint32_t *oy = S.out(out->y, groups * 16), *opk = S.out(out->pk, E * 16);
    uint8_t *ostatus = S.out(out->status, E), *ocomplete = S.out(out->complete, groups);
    uint64_t* obad = S.out(out->bad_actors, E);
    // NT = [N~; N~], H = [h1; h2; h1] (statement 1 is (N~, h1, h2), statement 2 (N~, h2, h1)), SEC = [phi - xhi; phi - xhi^-1],
    // RN = [r1; r2]: the two CompositeDLog proofs of every party run as one batch of 2E
    uint32_t *NT = S.tmp<uint32_t>(2 * E * 64), *H = S.tmp<uint32_t>(3 * E * 64), *SEC = S.tmp<uint32_t>(2 * E * 64), *RN = S.tmp<uint32_t>(2 * E * 16);
    uint32_t *X = S.tmp<uint32_t>(2 * E * 64), *Y = S.tmp<uint32_t>(2 * E * CDL_Y_LIMBS), *sigma = S.tmp<uint32_t>(E * 11 * 64);
    uint32_t *coeff = S.tmp<uint32_t>(E * t1 * 8), *shares = S.tmp<uint32_t>(E * (size_t)n * 8), *com = S.tmp<uint32_t>(E * 8);
    uint32_t *proof = S.tmp<uint32_t>(E * 40), *gcomm = S.tmp<uint32_t>(groups * (size_t)t1 * 16);
    uint8_t *st_nt = S.tmp<uint8_t>(E), *st_ckp = S.tmp<uint8_t>(E), *st_ck = S.tmp<uint8_t>(E), *st_cd = S.tmp<uint8_t>(2 * E), *ok2 = S.tmp<uint8_t>(E);
    uint8_t *pair_ok = S.tmp<uint8_t>(E * (size_t)n), *ok4 = S.tmp<uint8_t>(E), *salt = S.tmp<uint8_t>(sizeof(KEYGEN_SALT));
    if (S.err) return S.err;
    const cudaStream_t st = c->stream;
    if (cudaMemcpyAsync(salt, KEYGEN_SALT, sizeof(KEYGEN_SALT), cudaMemcpyHostToDevice, st) != cudaSuccess ||
        cudaMemcpyAsync(H, dh1, E * R, cudaMemcpyDeviceToDevice, st) != cudaSuccess ||
        cudaMemcpyAsync(H + 2 * E * 64, dh1, E * R, cudaMemcpyDeviceToDevice, st) != cudaSuccess ||
        cudaMemcpy2DAsync(RN, 16 * 4, dcdl, 32 * 4, 16 * 4, E, cudaMemcpyDeviceToDevice, st) != cudaSuccess ||
        cudaMemcpy2DAsync(RN + E * 16, 16 * 4, dcdl + 16, 32 * 4, 16 * 4, E, cudaMemcpyDeviceToDevice, st) != cudaSuccess ||
        cudaMemcpy2DAsync(coeff, t1 * 32, du, 32, 32, E, cudaMemcpyDeviceToDevice, st) != cudaSuccess ||
        cudaMemcpy2DAsync(coeff + 8, t1 * 32, da, t * 32, t * 32, E, cudaMemcpyDeviceToDevice, st) != cudaSuccess)
        return tecdsa_fail(TECDSA_E_CUDA, "gg20_keygen: copy");
    // Round 0 / 1: Keys::create and phase1_broadcast_phase3_proof_of_correct_key_proof_of_correct_h1h2 (party_i.rs:137-258)
    RUN(h1_h2_n_tilde_step(c, S, e, dpt, dqt, H, dxhi, NT, H + E * 64, SEC, SEC + E * 64, st_nt));
    if (cudaMemcpyAsync(NT + E * 64, NT, E * R, cudaMemcpyDeviceToDevice, st) != cudaSuccess) return tecdsa_fail(TECDSA_E_CUDA, "gg20_keygen: copy");
    // the prover's NOT_INVERTIBLE (no N^-1 mod phi) is not read: its exponent is then 0, every sigma is 1, and the
    // Round-2 NiCorrectKeyProof verification rejects that sender, as the reference's verifiers would reject its broadcast
    RUN(correct_key_prove_step(c, S, e, dp, dq, salt, (int)sizeof(KEYGEN_SALT), sigma, st_ckp, oN));
    RUN(composite_dlog_prove_step(c, 2 * e, NT, H, H + E * 64, SEC, 64, RN, X, Y, CDL_Y_LIMBS));
    RUN(vss_share_step(c, e, t1, n, coeff, shares, ovss));
    kg::k_kg_commit<<<grid_for(E), 64, 0, st>>>(ovss, t1, dblind, com, e);
    KCHECK();
    // Round 2 (party_i.rs:266-320), once per sender.  Here the decommitted y_i IS the sender's commitment 0 (ovss row 0) and com was
    // made above from the same y_i and blind, so the reopening check, like Round 3's commitments[0] == y_j, is a self-consistency
    // check of this call: it cannot fail here, and it is kept so that the kernels run every check the reference runs
    RUN(correct_key_verify_step(c, S, e, oN, sigma, salt, (int)sizeof(KEYGEN_SALT), st_ck));
    RUN(composite_dlog_verify_step(c, S, 2 * e, NT, H, H + E * 64, X, Y, CDL_Y_LIMBS, st_cd));
    kg::k_kg_round2<<<grid_for(E), 64, 0, st>>>(ovss, t1 * 16, dblind, com, st_ck, oN, NT, st_cd, ok2, e);
    KCHECK();
    // Round 3 (party_i.rs:322-367): every (receiver, sender) share, x_i, the DLog proof of x_i
    kg::k_kg_validate_pairs<<<grid_for(E * n), 64, 0, st>>>(ovss, t1, ovss, t1 * 16, shares, n, pair_ok, e * n);
    KCHECK();
    kg::k_kg_xi<<<grid_for(E), 64, 0, st>>>(shares, n, ox, e);
    KCHECK();
    kg::k_kg_dlog_prove<<<grid_for(E), 64, 0, st>>>(ox, ddl, proof, e);
    KCHECK();
    // Round 4 (party_i.rs:369-438), once per sender
    kg::k_kg_global_commitments<<<grid_for(groups * t1), 64, 0, st>>>(ovss, t1, n, gcomm, (int)groups);
    KCHECK();
    kg::k_kg_round4<<<grid_for(E), 64, 0, st>>>(gcomm, t1, n, proof, ok4, e);
    KCHECK();
    // LocalKey (keygen/rounds.rs:282-296): h1_h2_n_tilde_vec rows (N~, h1, h2), then status, masks, completion
    for (int k = 0; k < 3; k++)
        if (cudaMemcpy2DAsync(ost + k * 64, 3 * R, (k ? H + (k - 1) * E * 64 : NT), R, R, E, cudaMemcpyDeviceToDevice, st) != cudaSuccess)
            return tecdsa_fail(TECDSA_E_CUDA, "gg20_keygen: copy");
    kg::k_kg_finish<<<grid_for(E), 64, 0, st>>>(n, t1, st_nt, ok2, pair_ok, ok4, proof, gcomm, ostatus, obad, ocomplete, opk, oy, ox, ovss, oN, ost, e);
    KCHECK();
    return S.finish();
}
