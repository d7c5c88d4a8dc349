// L0 surface of curv-kzen `Scalar<Secp256k1>` / `Point<Secp256k1>` / `BigInt` that is not a modular exponentiation, batched:
// the operators and helpers src/protocols/* and src/utilities/* call between the heavy steps
// (/root/reference/src/protocols/multi_party_ecdsa/gg_2020/party_i.rs:559-563,599-617,627-639,771-772,857-863,914-929;
//  src/utilities/mta/range_proofs.rs:87-88,538-557).  One thread per element; the device functions are those of the offline
// stage (secp256k1.cuh, st_bigint.cuh, sha256.cuh), so a value computed here is the value the L3 driver computes.
#include "stage.cuh"

using namespace tecdsa;

int tecdsa_internal_fb_points_set_ecops(const uint32_t* table) {
    CK(cudaMemcpyToSymbol(secp::g_fb_points, &table, sizeof(table)));
    return 0;
}

namespace {

// op: 0 = a + b, 1 = a - b   (`Point + Point`, `Point - Point`; party_i.rs:771-772, 839-840)
__global__ void k_pt_addsub(const uint32_t* a, const uint32_t* b, uint32_t* out, int op, int count) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    Affine pa = affine_load(a + (size_t)i * 16), pb = affine_load(b + (size_t)i * 16);
    Jac jb = jac_from_affine(pb);
    if (op) jb = jac_neg(jb);
    affine_store(out + (size_t)i * 16, jac_to_affine(jac_add(jac_from_affine(pa), jb)));
}
// `Point::to_bytes(true)`: 33 bytes SEC1; the identity encodes as 33 zero bytes here (curv: a single 0x00)
__global__ void k_pt_compress(const uint32_t* pts, uint8_t* out33, int count) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    Affine p = affine_load(pts + (size_t)i * 16);
    uint8_t* o = out33 + (size_t)i * 33;
    if (p.inf) { for (int k = 0; k < 33; k++) o[k] = 0; return; }
    affine_compress(o, p);
}
// `Point::from_bytes` of a 33-byte compressed encoding: y = sqrt(x^3 + 7) with the requested parity; ok = 0 for x >= p, a
// non-residue, or a bad prefix byte (curv: DeserializationError)
__global__ void k_pt_decompress(const uint8_t* in33, uint32_t* pts, uint8_t* ok, int count) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    const uint8_t* b = in33 + (size_t)i * 33;
    U256 x = u256_zero();
    for (int k = 0; k < 32; k++) x.v[7 - (k >> 2)] |= (uint32_t)b[1 + k] << (8 * (3 - (k & 3)));
    bool good = (b[0] == 2 || b[0] == 3) && !u256_ge(x, P_LIMBS);
    U256 seven = u256_zero(); seven.v[0] = 7;
    const U256 rhs = fe_add(fe_mul(fe_sqr(x), x), seven);
    // p = 3 mod 4: sqrt = rhs^((p+1)/4), (p+1)/4 = 2^254 - 2^30 - 244
    U256 e = u256_zero();
    for (int k = 0; k < 8; k++) e.v[k] = 0xFFFFFFFFu;
    e.v[7] = 0x3FFFFFFFu; e.v[0] = 0xBFFFFF0Cu;
    U256 y = u256_one();
    for (int bit = 253; bit >= 0; bit--) {
        y = fe_sqr(y);
        if ((e.v[bit >> 5] >> (bit & 31)) & 1u) y = fe_mul(y, rhs);
    }
    good = good && u256_eq(fe_sqr(y), rhs);
    if ((y.v[0] & 1u) != (uint32_t)(b[0] & 1u)) y = fe_neg(y);
    uint32_t* o = pts + (size_t)i * 16;
    if (!good) { for (int k = 0; k < 16; k++) o[k] = 0; }
    else { u256_store(o, x); u256_store(o + 8, y); }
    ok[i] = good ? 1 : 0;
}
// op: 0 = a*b, 1 = a+b, 2 = a-b, 3 = a^-1 (b unused; ok = 0 for a == 0, `Scalar::invert` -> None) — all mod q
__global__ void k_scalar_op(const uint32_t* a, const uint32_t* b, uint32_t* out, uint8_t* ok, int op, int count) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    const U256 x = load_scalar(a + (size_t)i * 8);
    U256 r;
    bool good = true;
    if (op == 3) { good = !u256_is_zero(x); r = good ? sc_inv(x) : u256_zero(); }
    else {
        const U256 y = load_scalar(b + (size_t)i * 8);
        r = op == 0 ? sc_mul(x, y) : op == 1 ? sc_add(x, y) : sc_sub(x, y);
    }
    u256_store(out + (size_t)i * 8, r);
    if (ok) ok[i] = good ? 1 : 0;
}
// `Scalar::from(&BigInt)`: any non-negative integer of `limbs` limbs reduced mod q
__global__ void k_scalar_from(const uint32_t* x, int limbs, uint32_t* out, int count) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    u256_store(out + (size_t)i * 8, sc_from_limbs(x + (size_t)i * limbs, limbs));
}
// exact a*b + c over the integers (`e * a + alpha`, range_proofs.rs:87-88)
__global__ void k_wide_muladd(const uint32_t* a, int al, const uint32_t* b, int bl, const uint32_t* c, int cl, uint32_t* out, int ol, int count) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    st::mul_add(out + (size_t)i * ol, ol, a + (size_t)i * al, al, b + (size_t)i * bl, bl, c + (size_t)i * cl, cl);
}
// the acceptance test of `SampleFromMultiplicativeGroup::from_modulo` (range_proofs.rs:543-552): r < N (sample_below) and
// gcd(r, N) == 1 (inv_ok of the inversion job)
__global__ void k_unit_check(const uint32_t* r, const uint32_t* n, const uint32_t* idx, int K, const uint8_t* inv_ok, uint8_t* ok, int count) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    const uint32_t* m = n + (size_t)(idx ? idx[i] : (uint32_t)i) * K;
    ok[i] = (inv_ok[i] && st::cmp(r + (size_t)i * K, m, K) < 0) ? 1 : 0;
}
// SHA-256 of arbitrary byte strings: message i = bytes[offsets[i] .. offsets[i+1])
__global__ void k_sha256_bytes(const uint8_t* bytes, const uint64_t* offsets, uint8_t* out32, int count) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    Sha256 h; h.init();
    for (uint64_t p = offsets[i]; p < offsets[i + 1]; p++) h.put(bytes[p]);
    uint32_t d[8];
    h.finish(d);
    for (int k = 0; k < 32; k++) out32[(size_t)i * 32 + k] = (uint8_t)(d[7 - (k >> 2)] >> (8 * (3 - (k & 3))));
}

}  // namespace

static int pt_addsub(tecdsa_ctx* c, const uint32_t* a, const uint32_t* b, uint32_t* out, int op, size_t count, int mem, const char* name) {
    if (!a || !b || !out) return tecdsa_fail(TECDSA_E_ARG, name);
    STAGE_PROLOGUE("secp point op", count);
    const uint32_t *da = S.in(a, count * 16), *db = S.in(b, count * 16);
    uint32_t* dout = S.out(out, count * 16);
    if (S.err) return S.err;
    k_pt_addsub<<<grid_for(count), 64, 0, c->stream>>>(da, db, dout, op, (int)count);
    KCHECK();
    return S.finish();
}
extern "C" int tecdsa_secp_add_batch(tecdsa_ctx* c, const uint32_t* a, const uint32_t* b, uint32_t* out, size_t count, int mem) {
    return pt_addsub(c, a, b, out, 0, count, mem, "secp_add: null argument");
}
extern "C" int tecdsa_secp_sub_batch(tecdsa_ctx* c, const uint32_t* a, const uint32_t* b, uint32_t* out, size_t count, int mem) {
    return pt_addsub(c, a, b, out, 1, count, mem, "secp_sub: null argument");
}
extern "C" int tecdsa_secp_compress_batch(tecdsa_ctx* c, const uint32_t* points, uint8_t* out33, size_t count, int mem) {
    if (!points || !out33) return tecdsa_fail(TECDSA_E_ARG, "secp_compress: null argument");
    STAGE_PROLOGUE("secp_compress", count);
    const uint32_t* dp = S.in(points, count * 16);
    uint8_t* dout = S.out(out33, count * 33);
    if (S.err) return S.err;
    k_pt_compress<<<grid_for(count), 64, 0, c->stream>>>(dp, dout, (int)count);
    KCHECK();
    return S.finish();
}
extern "C" int tecdsa_secp_decompress_batch(tecdsa_ctx* c, const uint8_t* in33, uint32_t* points, uint8_t* ok, size_t count, int mem) {
    if (!in33 || !points || !ok) return tecdsa_fail(TECDSA_E_ARG, "secp_decompress: null argument");
    STAGE_PROLOGUE("secp_decompress", count);
    const uint8_t* din = S.in(in33, count * 33);
    uint32_t* dp = S.out(points, count * 16);
    uint8_t* dok = S.out(ok, count);
    if (S.err) return S.err;
    k_pt_decompress<<<grid_for(count), 64, 0, c->stream>>>(din, dp, dok, (int)count);
    KCHECK();
    return S.finish();
}
static int scalar_op(tecdsa_ctx* c, const uint32_t* a, const uint32_t* b, uint32_t* out, uint8_t* ok, int op, size_t count, int mem) {
    if (!a || !out || (op != 3 && !b)) return tecdsa_fail(TECDSA_E_ARG, "secp scalar op: null argument");
    STAGE_PROLOGUE("secp scalar op", count);
    const uint32_t *da = S.in(a, count * 8), *db = S.in(b, count * 8);
    uint32_t* dout = S.out(out, count * 8);
    uint8_t* dok = S.out(ok, count);
    if (S.err) return S.err;
    k_scalar_op<<<grid_for(count), 64, 0, c->stream>>>(da, db, dout, dok, op, (int)count);
    KCHECK();
    return S.finish();
}
extern "C" int tecdsa_secp_scalar_mul_batch(tecdsa_ctx* c, const uint32_t* a, const uint32_t* b, uint32_t* out, size_t count, int mem) { return scalar_op(c, a, b, out, nullptr, 0, count, mem); }
extern "C" int tecdsa_secp_scalar_add_batch(tecdsa_ctx* c, const uint32_t* a, const uint32_t* b, uint32_t* out, size_t count, int mem) { return scalar_op(c, a, b, out, nullptr, 1, count, mem); }
extern "C" int tecdsa_secp_scalar_sub_batch(tecdsa_ctx* c, const uint32_t* a, const uint32_t* b, uint32_t* out, size_t count, int mem) { return scalar_op(c, a, b, out, nullptr, 2, count, mem); }
extern "C" int tecdsa_secp_scalar_inv_batch(tecdsa_ctx* c, const uint32_t* a, uint32_t* out, uint8_t* ok, size_t count, int mem) { return scalar_op(c, a, nullptr, out, ok, 3, count, mem); }
extern "C" int tecdsa_secp_scalar_from_bigint_batch(tecdsa_ctx* c, const uint32_t* x, int limbs, uint32_t* out, size_t count, int mem) {
    if (!x || !out || limbs <= 0 || limbs > 256) return tecdsa_fail(TECDSA_E_ARG, "secp_scalar_from_bigint: bad argument");
    STAGE_PROLOGUE("secp_scalar_from_bigint", count);
    const uint32_t* dx = S.in(x, count * (size_t)limbs);
    uint32_t* dout = S.out(out, count * 8);
    if (S.err) return S.err;
    k_scalar_from<<<grid_for(count), 64, 0, c->stream>>>(dx, limbs, dout, (int)count);
    KCHECK();
    return S.finish();
}
// The widths must make a*b + c fit in out_limbs for EVERY operand value (st::mul_add drops a carry out of the top limb):
// one limb above both a*b and c, or exactly a_limbs + b_limbs when c is no wider than the wider factor
// ((2^(32A) - 1)(2^(32B) - 1) + 2^(32 max(A,B)) - 1 < 2^(32(A+B))).
static bool wide_muladd_fits(int a_limbs, int b_limbs, int c_limbs, int out_limbs) {
    const int ab = a_limbs + b_limbs, wider = a_limbs > b_limbs ? a_limbs : b_limbs;
    return out_limbs >= (ab > c_limbs ? ab : c_limbs) + 1 || (out_limbs == ab && c_limbs <= wider);
}
extern "C" int tecdsa_wide_muladd_batch(tecdsa_ctx* c, const uint32_t* a, int a_limbs, const uint32_t* b, int b_limbs, const uint32_t* addend, int c_limbs,
                                        uint32_t* out, int out_limbs, size_t count, int mem) {
    if (!a || !b || !addend || !out || a_limbs <= 0 || b_limbs <= 0 || c_limbs <= 0 || out_limbs > 512 ||
        !wide_muladd_fits(a_limbs, b_limbs, c_limbs, out_limbs))
        return tecdsa_fail(TECDSA_E_ARG, "wide_muladd: bad argument (out_limbs must hold a*b + c for all operand values)");
    STAGE_PROLOGUE("wide_muladd", count);
    const uint32_t *da = S.in(a, count * (size_t)a_limbs), *db = S.in(b, count * (size_t)b_limbs), *dc = S.in(addend, count * (size_t)c_limbs);
    uint32_t* dout = S.out(out, count * (size_t)out_limbs);
    if (S.err) return S.err;
    k_wide_muladd<<<grid_for(count), 64, 0, c->stream>>>(da, a_limbs, db, b_limbs, dc, c_limbs, dout, out_limbs, (int)count);
    KCHECK();
    return S.finish();
}
extern "C" int tecdsa_unit_mod_check_batch(tecdsa_ctx* c, int mod_bits, const uint32_t* r, const uint32_t* modulus, const uint32_t* mod_idx, size_t n_mod,
                                           uint8_t* ok, size_t count, int mem) {
    if (!r || !modulus || !ok) return tecdsa_fail(TECDSA_E_ARG, "unit_mod_check: null argument");
    if (check_bits(mod_bits)) return TECDSA_E_UNSUPPORTED;
    STAGE_PROLOGUE("unit_mod_check", count);
    const int n = (int)count;
    const int K = mod_bits / 32;
    const uint32_t *dr = S.in(r, count * K), *dm = S.in(modulus, (mod_idx ? n_mod : count) * K), *di = S.in(mod_idx, count);
    uint8_t* dok = S.out(ok, count);
    uint32_t* scratch = S.tmp<uint32_t>(count * K);
    uint8_t* inv_ok = S.tmp<uint8_t>(count);
    if (S.err) return S.err;
    Launches L;
    InvLaunch& l = K == 64 ? L.i64 : L.i128;
    add_inv(l, K, n, di ? tab(dm, di, K) : arr(dm, K), arr(dr, K), scratch, inv_ok);
    RUN(run(c, l, K));
    k_unit_check<<<grid_for(count), 64, 0, c->stream>>>(dr, dm, di, K, inv_ok, dok, n);
    KCHECK();
    return S.finish();
}
extern "C" int tecdsa_sha256_batch(tecdsa_ctx* c, const uint8_t* bytes, const uint64_t* offsets, uint8_t* digests, size_t count, int mem) {
    if (!offsets || !digests) return tecdsa_fail(TECDSA_E_ARG, "sha256: null argument");
    if (mem != TECDSA_HOST) return tecdsa_fail(TECDSA_E_UNSUPPORTED, "sha256: the offsets array is read on the host to size the copy; pass TECDSA_HOST buffers");
    STAGE_PROLOGUE("sha256", count);
    const size_t total = offsets[count];
    for (size_t i = 0; i < count; i++) if (offsets[i] > offsets[i + 1]) return tecdsa_fail(TECDSA_E_ARG, "sha256: offsets must not decrease");
    if (total && !bytes) return tecdsa_fail(TECDSA_E_ARG, "sha256: null message buffer");
    const uint8_t* db = S.in(bytes, total ? total : 1);
    const uint64_t* doff = S.in(offsets, count + 1);
    uint8_t* dout = S.out(digests, count * 32);
    if (S.err) return S.err;
    k_sha256_bytes<<<grid_for(count), 64, 0, c->stream>>>(db, doff, dout, (int)count);
    KCHECK();
    return S.finish();
}
