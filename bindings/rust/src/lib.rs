//! Rust shim over the C ABI of the engine (`include/tecdsa_b200.h`).
//!
//! The reference (ZenGo-X/multi-party-ecdsa @ 7d8bd41) has no FFI: its seam is the trait surface of curv-kzen `BigInt`,
//! `Scalar<Secp256k1>` / `Point<Secp256k1>`, kzen-paillier `Paillier::*` and the in-tree proof structs.  This crate gives that
//! surface two forms:
//!   * `scalar`: drop-in, batch-of-1 equivalents of the scalar calls the protocol code makes (`mod_pow`, `mod_inv`,
//!     `Paillier::encrypt_with_chosen_randomness`, `Point * Scalar`, ...) — correct, but one PCIe round trip per call;
//!   * `batch`: the calls as the engine wants them, a whole batch of independent instances per call (proof generation /
//!     verification, the offline stage, the online step).
//! `ffi` is generated from the header (tools/gen_rust_ffi.py) and lists every exported symbol.
//!
//! NOT compiled in the development image (no cargo/rustc, crates not vendored): treat it as the maintainer's starting point.
pub mod ffi;

use curv::arithmetic::traits::*;
use curv::elliptic::curves::{Point, Scalar, Secp256k1};
use curv::BigInt;
use std::os::raw::c_int;
use std::ptr;

#[derive(Debug)]
pub struct EngineError(pub c_int, pub String);

fn check(rc: c_int) -> Result<(), EngineError> {
    if rc == 0 {
        return Ok(());
    }
    let msg = unsafe { std::ffi::CStr::from_ptr(ffi::tecdsa_last_error()) }.to_string_lossy().into_owned();
    Err(EngineError(rc, msg))
}

/// One engine context = one GPU + one stream (`tecdsa_ctx`).  Not `Sync`: a context is single-threaded by contract.
pub struct Engine {
    ctx: *mut ffi::tecdsa_ctx,
}

impl Engine {
    pub fn new(device: i32) -> Result<Self, EngineError> {
        let mut ctx = ptr::null_mut();
        check(unsafe { ffi::tecdsa_ctx_create(&mut ctx, device, ptr::null_mut()) })?;
        Ok(Engine { ctx })
    }
    pub fn raw(&self) -> *mut ffi::tecdsa_ctx {
        self.ctx
    }
}
impl Drop for Engine {
    fn drop(&mut self) {
        unsafe { ffi::tecdsa_ctx_destroy(self.ctx) };
    }
}

// ---------------------------------------------------------------------------------------------- limb packing
/// `BigInt` -> `k` little-endian u32 limbs (the ABI's operand layout); panics if the value does not fit or is negative.
pub fn to_limbs(x: &BigInt, k: usize) -> Vec<u32> {
    assert!(x >= &BigInt::zero(), "negative BigInt at the FFI boundary");
    let bytes = x.to_bytes(); // big-endian magnitude
    assert!(bytes.len() <= 4 * k, "BigInt wider than {} limbs", k);
    let mut out = vec![0u32; k];
    for (i, b) in bytes.iter().rev().enumerate() {
        out[i / 4] |= (*b as u32) << (8 * (i % 4));
    }
    out
}
pub fn from_limbs(l: &[u32]) -> BigInt {
    let mut bytes = Vec::with_capacity(4 * l.len());
    for w in l.iter().rev() {
        bytes.extend_from_slice(&w.to_be_bytes());
    }
    BigInt::from_bytes(&bytes)
}
/// affine point -> x||y (16 limbs, all-zero = identity)
pub fn point_to_limbs(p: &Point<Secp256k1>) -> Vec<u32> {
    match (p.x_coord(), p.y_coord()) {
        (Some(x), Some(y)) => {
            let mut v = to_limbs(&x, 8);
            v.extend(to_limbs(&y, 8));
            v
        }
        _ => vec![0u32; 16],
    }
}
pub fn point_from_limbs(l: &[u32]) -> Point<Secp256k1> {
    if l.iter().all(|w| *w == 0) {
        return Point::zero();
    }
    Point::from_coords(&from_limbs(&l[..8]), &from_limbs(&l[8..16])).expect("engine returned a point off the curve")
}
pub fn scalar_to_limbs(s: &Scalar<Secp256k1>) -> Vec<u32> {
    to_limbs(&s.to_bigint(), 8)
}
pub fn scalar_from_limbs(l: &[u32]) -> Scalar<Secp256k1> {
    Scalar::from(&from_limbs(l))
}

// ---------------------------------------------------------------------------------------------- batch-of-1 scalar surface
/// The scalar calls of `curv::arithmetic::traits::{Modulo, ...}`, `Point * Scalar` and `Paillier::*` as batch-of-1 engine
/// calls.  Semantics are those of the reference: `mod_inv` returns `None` when gcd != 1, results are canonical residues.
pub mod scalar {
    use super::*;

    fn width(m: &BigInt) -> (c_int, usize) {
        if m.bit_length() <= 2048 { (2048, 64) } else { (4096, 128) }
    }
    /// `BigInt::mod_pow(base, exponent, modulus)` — odd moduli up to 4096 bits (utilities/mta/range_proofs.rs:52)
    pub fn mod_pow(e: &Engine, base: &BigInt, exponent: &BigInt, modulus: &BigInt) -> Result<BigInt, EngineError> {
        let (bits, k) = width(modulus);
        let el = ((exponent.bit_length() + 31) / 32).max(1);
        let (b, x, m) = (to_limbs(&base.modulus(modulus), k), to_limbs(exponent, el), to_limbs(modulus, k));
        let mut out = vec![0u32; k];
        let mut st = [0u8; 1];
        check(unsafe {
            ffi::tecdsa_modexp_batch(e.raw(), bits, el as c_int, b.as_ptr(), x.as_ptr(), m.as_ptr(), ptr::null(), 0, out.as_mut_ptr(), st.as_mut_ptr(), 1, ffi::TECDSA_HOST)
        })?;
        if st[0] != 0 {
            return Err(EngineError(st[0] as c_int, "even modulus".into()));
        }
        Ok(from_limbs(&out))
    }
    /// `BigInt::mod_mul`
    pub fn mod_mul(e: &Engine, a: &BigInt, b: &BigInt, modulus: &BigInt) -> Result<BigInt, EngineError> {
        let (bits, k) = width(modulus);
        let (x, y, m) = (to_limbs(&a.modulus(modulus), k), to_limbs(&b.modulus(modulus), k), to_limbs(modulus, k));
        let mut out = vec![0u32; k];
        check(unsafe { ffi::tecdsa_modmul_batch(e.raw(), bits, x.as_ptr(), y.as_ptr(), m.as_ptr(), ptr::null(), 0, out.as_mut_ptr(), 1, ffi::TECDSA_HOST) })?;
        Ok(from_limbs(&out))
    }
    /// `BigInt::mod_inv -> Option<BigInt>`
    pub fn mod_inv(e: &Engine, a: &BigInt, modulus: &BigInt) -> Result<Option<BigInt>, EngineError> {
        let (bits, k) = width(modulus);
        let (x, m) = (to_limbs(&a.modulus(modulus), k), to_limbs(modulus, k));
        let mut out = vec![0u32; k];
        let mut ok = [0u8; 1];
        check(unsafe { ffi::tecdsa_modinv_batch(e.raw(), bits, x.as_ptr(), m.as_ptr(), ptr::null(), 0, out.as_mut_ptr(), ok.as_mut_ptr(), 1, ffi::TECDSA_HOST) })?;
        Ok(if ok[0] == 1 { Some(from_limbs(&out)) } else { None })
    }
    /// `r.gcd(N) == 1 && r < N` — the loop condition of `SampleFromMultiplicativeGroup` (utilities/mta/range_proofs.rs:543-552)
    pub fn is_unit_below(e: &Engine, r: &BigInt, n: &BigInt) -> Result<bool, EngineError> {
        let (bits, k) = width(n);
        if r.bit_length() > 32 * k { return Ok(false); }
        let (x, m) = (to_limbs(r, k), to_limbs(n, k));
        let mut ok = [0u8; 1];
        check(unsafe { ffi::tecdsa_unit_mod_check_batch(e.raw(), bits, x.as_ptr(), m.as_ptr(), ptr::null(), 0, ok.as_mut_ptr(), 1, ffi::TECDSA_HOST) })?;
        Ok(ok[0] == 1)
    }
    /// `Point * Scalar`; `point == None` is `Point::generator() * s` (gg_2020/party_i.rs:560-562,682,784)
    pub fn point_mul(e: &Engine, point: Option<&Point<Secp256k1>>, s: &Scalar<Secp256k1>) -> Result<Point<Secp256k1>, EngineError> {
        let k = scalar_to_limbs(s);
        let p = point.map(point_to_limbs);
        let mut out = vec![0u32; 16];
        check(unsafe { ffi::tecdsa_secp_mul_batch(e.raw(), p.as_ref().map_or(ptr::null(), |v| v.as_ptr()), k.as_ptr(), out.as_mut_ptr(), 1, ffi::TECDSA_HOST) })?;
        Ok(point_from_limbs(&out))
    }
    /// `Point + Point`
    pub fn point_add(e: &Engine, a: &Point<Secp256k1>, b: &Point<Secp256k1>) -> Result<Point<Secp256k1>, EngineError> {
        let (x, y) = (point_to_limbs(a), point_to_limbs(b));
        let mut out = vec![0u32; 16];
        check(unsafe { ffi::tecdsa_secp_add_batch(e.raw(), x.as_ptr(), y.as_ptr(), out.as_mut_ptr(), 1, ffi::TECDSA_HOST) })?;
        Ok(point_from_limbs(&out))
    }
    /// `Point::to_bytes(true)`
    pub fn point_to_bytes(e: &Engine, p: &Point<Secp256k1>) -> Result<[u8; 33], EngineError> {
        let x = point_to_limbs(p);
        let mut out = [0u8; 33];
        check(unsafe { ffi::tecdsa_secp_compress_batch(e.raw(), x.as_ptr(), out.as_mut_ptr(), 1, ffi::TECDSA_HOST) })?;
        Ok(out)
    }
    /// `Scalar * Scalar`, `+`, `-`, `invert()` (gg_2020/party_i.rs:599-617,635-640,857-863)
    pub fn scalar_mul(e: &Engine, a: &Scalar<Secp256k1>, b: &Scalar<Secp256k1>) -> Result<Scalar<Secp256k1>, EngineError> {
        let (x, y) = (scalar_to_limbs(a), scalar_to_limbs(b));
        let mut out = vec![0u32; 8];
        check(unsafe { ffi::tecdsa_secp_scalar_mul_batch(e.raw(), x.as_ptr(), y.as_ptr(), out.as_mut_ptr(), 1, ffi::TECDSA_HOST) })?;
        Ok(scalar_from_limbs(&out))
    }
    pub fn scalar_invert(e: &Engine, a: &Scalar<Secp256k1>) -> Result<Option<Scalar<Secp256k1>>, EngineError> {
        let x = scalar_to_limbs(a);
        let mut out = vec![0u32; 8];
        let mut ok = [0u8; 1];
        check(unsafe { ffi::tecdsa_secp_scalar_inv_batch(e.raw(), x.as_ptr(), out.as_mut_ptr(), ok.as_mut_ptr(), 1, ffi::TECDSA_HOST) })?;
        Ok(if ok[0] == 1 { Some(scalar_from_limbs(&out)) } else { None })
    }
    /// `Paillier::encrypt_with_chosen_randomness(ek, RawPlaintext(m), &Randomness(r))` (utilities/mta/mod.rs:68,133)
    pub fn paillier_encrypt(e: &Engine, n: &BigInt, m: &BigInt, r: &BigInt) -> Result<BigInt, EngineError> {
        let (nl, ml, rl) = (to_limbs(n, 64), to_limbs(m, 64), to_limbs(r, 64));
        let mut c = vec![0u32; 128];
        check(unsafe { ffi::tecdsa_paillier_encrypt_batch(e.raw(), nl.as_ptr(), ptr::null(), 1, ml.as_ptr(), rl.as_ptr(), c.as_mut_ptr(), 1, ffi::TECDSA_HOST) })?;
        Ok(from_limbs(&c))
    }
    /// `Paillier::mul(ek, c, k)` = c^k mod n^2 (utilities/mta/mod.rs:140)
    pub fn paillier_mul(e: &Engine, n: &BigInt, c: &BigInt, k: &BigInt) -> Result<BigInt, EngineError> {
        let kl = ((k.bit_length() + 127) / 128 * 4).max(4);
        let (nl, cl, kk) = (to_limbs(n, 64), to_limbs(c, 128), to_limbs(k, kl));
        let mut out = vec![0u32; 128];
        check(unsafe { ffi::tecdsa_paillier_mul_batch(e.raw(), nl.as_ptr(), ptr::null(), 1, cl.as_ptr(), kk.as_ptr(), kl as c_int, out.as_mut_ptr(), 1, ffi::TECDSA_HOST) })?;
        Ok(from_limbs(&out))
    }
    /// `Paillier::add(ek, c1, c2)` = c1 c2 mod n^2 (utilities/mta/mod.rs:145)
    pub fn paillier_add(e: &Engine, n: &BigInt, c1: &BigInt, c2: &BigInt) -> Result<BigInt, EngineError> {
        let (nl, a, b) = (to_limbs(n, 64), to_limbs(c1, 128), to_limbs(c2, 128));
        let mut out = vec![0u32; 128];
        check(unsafe { ffi::tecdsa_paillier_add_batch(e.raw(), nl.as_ptr(), ptr::null(), 1, a.as_ptr(), b.as_ptr(), out.as_mut_ptr(), 1, ffi::TECDSA_HOST) })?;
        Ok(from_limbs(&out))
    }
}

// ---------------------------------------------------------------------------------------------- key sets + batched calls
/// Device-resident `LocalKey` material of `n_keysets` (t = 1, n = 3) key sets: rows are `keyset * 3 + party`.
pub struct KeySets {
    ks: *mut ffi::tecdsa_keyset,
    ctx: *mut ffi::tecdsa_ctx,
}
pub struct PartyKey<'a> {
    pub p: &'a BigInt,
    pub q: &'a BigInt,
    pub n_tilde: &'a BigInt,
    pub h1: &'a BigInt,
    pub h2: &'a BigInt,
    pub x_i: &'a Scalar<Secp256k1>,
    pub pk: &'a Point<Secp256k1>,
}
impl KeySets {
    /// `parties` = 3 entries per key set (keygen indices 1..3), `y` = one public key per key set
    pub fn upload(e: &Engine, parties: &[PartyKey], y: &[Point<Secp256k1>]) -> Result<Self, EngineError> {
        assert_eq!(parties.len(), 3 * y.len());
        let cat = |f: &dyn Fn(&PartyKey) -> Vec<u32>| parties.iter().flat_map(|p| f(p)).collect::<Vec<u32>>();
        let (p, q) = (cat(&|k| to_limbs(k.p, 32)), cat(&|k| to_limbs(k.q, 32)));
        let (nt, h1, h2) = (cat(&|k| to_limbs(k.n_tilde, 64)), cat(&|k| to_limbs(k.h1, 64)), cat(&|k| to_limbs(k.h2, 64)));
        let (x, pk) = (cat(&|k| scalar_to_limbs(k.x_i)), cat(&|k| point_to_limbs(k.pk)));
        let yl: Vec<u32> = y.iter().flat_map(point_to_limbs).collect();
        let keys = ffi::tecdsa_keys { n_keysets: y.len(), paillier_p: p.as_ptr(), paillier_q: q.as_ptr(), n_tilde: nt.as_ptr(), h1: h1.as_ptr(), h2: h2.as_ptr(),
                                      x_i: x.as_ptr(), pk: pk.as_ptr(), y: yl.as_ptr() };
        let mut ks = ptr::null_mut();
        check(unsafe { ffi::tecdsa_keys_upload(e.raw(), &keys, &mut ks) })?;
        Ok(KeySets { ks, ctx: e.raw() })
    }
    pub fn raw(&self) -> *mut ffi::tecdsa_keyset {
        self.ks
    }
}
impl Drop for KeySets {
    fn drop(&mut self) {
        unsafe { ffi::tecdsa_keys_free(self.ctx, self.ks) };
    }
}

pub mod batch {
    use super::*;

    /// The public fields of `AliceProof` (the reference keeps them private; its serde form is the interchange format)
    #[derive(Clone, Debug)]
    pub struct AliceProofParts { pub z: BigInt, pub e: BigInt, pub s: BigInt, pub s1: BigInt, pub s2: BigInt }

    /// `AliceProof::verify(&cipher, &ek, &dlog_statement)` for a batch (utilities/mta/range_proofs.rs:105-156): one bool per proof
    pub fn alice_proof_verify(e: &Engine, ks: &KeySets, ek_row: &[u32], st_row: &[u32], cipher: &[BigInt], proofs: &[AliceProofParts]) -> Result<Vec<bool>, EngineError> {
        let n = proofs.len();
        assert!(ek_row.len() == n && st_row.len() == n && cipher.len() == n);
        // a field wider than its slot can never verify (s1 > q^3, s2 > q N~ ...): reject it here instead of truncating
        let fits = |x: &BigInt, limbs: usize| x >= &BigInt::zero() && x.bit_length() <= 32 * limbs;
        let bad: Vec<bool> = proofs.iter().map(|p| !(fits(&p.z, 64) && fits(&p.e, 8) && fits(&p.s, 64) && fits(&p.s1, 28) && fits(&p.s2, 92))).collect();
        let zero = BigInt::zero();
        let col = |f: &dyn Fn(&AliceProofParts) -> &BigInt, limbs: usize| -> Vec<u32> {
            proofs.iter().zip(&bad).flat_map(|(p, b)| to_limbs(if *b { &zero } else { f(p) }, limbs)).collect()
        };
        let c: Vec<u32> = cipher.iter().flat_map(|x| to_limbs(x, 128)).collect();
        let (z, ee, s, s1, s2) = (col(&|p| &p.z, 64), col(&|p| &p.e, 8), col(&|p| &p.s, 64), col(&|p| &p.s1, 28), col(&|p| &p.s2, 92));
        let mut st = vec![255u8; n];
        check(unsafe {
            ffi::tecdsa_alice_proof_verify_batch(e.raw(), ks.raw(), ek_row.as_ptr(), st_row.as_ptr(), c.as_ptr(), z.as_ptr(), ee.as_ptr(), s.as_ptr(), s1.as_ptr(),
                                                 s2.as_ptr(), st.as_mut_ptr(), n, ffi::TECDSA_HOST)
        })?;
        Ok(st.iter().zip(&bad).map(|(s, b)| *s == 0 && !*b).collect())
    }

    /// `AliceProof::generate(a, cipher, ek, dlog_statement, r)` with the four sampled values explicit (range_proofs.rs:160-193)
    #[allow(clippy::too_many_arguments)]
    pub fn alice_proof_generate(e: &Engine, ks: &KeySets, ek_row: &[u32], st_row: &[u32], a: &[BigInt], cipher: &[BigInt], r: &[BigInt],
                                alpha: &[BigInt], beta: &[BigInt], gamma: &[BigInt], rho: &[BigInt]) -> Result<Vec<AliceProofParts>, EngineError> {
        let n = a.len();
        let pack = |v: &[BigInt], limbs: usize| -> Vec<u32> { v.iter().flat_map(|x| to_limbs(x, limbs)).collect() };
        let (al, cl, rl, alp, bet, gam, rh) = (pack(a, 8), pack(cipher, 128), pack(r, 64), pack(alpha, 24), pack(beta, 64), pack(gamma, 88), pack(rho, 72));
        let (mut z, mut ee, mut s, mut s1, mut s2) = (vec![0u32; n * 64], vec![0u32; n * 8], vec![0u32; n * 64], vec![0u32; n * 28], vec![0u32; n * 92]);
        check(unsafe {
            ffi::tecdsa_alice_proof_generate_batch(e.raw(), ks.raw(), ek_row.as_ptr(), st_row.as_ptr(), al.as_ptr(), cl.as_ptr(), rl.as_ptr(), alp.as_ptr(), bet.as_ptr(),
                                                   gam.as_ptr(), rh.as_ptr(), z.as_mut_ptr(), ee.as_mut_ptr(), s.as_mut_ptr(), s1.as_mut_ptr(), s2.as_mut_ptr(), n, ffi::TECDSA_HOST)
        })?;
        Ok((0..n).map(|i| AliceProofParts { z: from_limbs(&z[i * 64..(i + 1) * 64]), e: from_limbs(&ee[i * 8..(i + 1) * 8]), s: from_limbs(&s[i * 64..(i + 1) * 64]),
                                            s1: from_limbs(&s1[i * 28..(i + 1) * 28]), s2: from_limbs(&s2[i * 92..(i + 1) * 92]) }).collect())
    }

    /// The batched `OfflineStage` (sign/rounds.rs:68-636): `sessions[s] = [keyset, party0, party1]`, `rnd` = `2 * sessions.len()`
    /// randomness records of `ffi::TECDSA_RND_LIMBS` limbs (layout: `TECDSA_RND_*` in the header).  Returns the 256-byte
    /// result records (`TECDSA_REC_*`), one per unit.
    pub fn offline_records(e: &Engine, ks: &KeySets, sessions: &[[u32; 3]], rnd: &[u32]) -> Result<Vec<u8>, EngineError> {
        let n = sessions.len();
        assert_eq!(rnd.len(), 2 * n * ffi::TECDSA_RND_LIMBS);
        let flat: Vec<u32> = sessions.iter().flat_map(|s| s.iter().copied()).collect();
        let mut rec = vec![0u8; 2 * n * ffi::TECDSA_REC_BYTES];
        check(unsafe { ffi::tecdsa_gg20_offline_records(e.raw(), ks.raw(), ptr::null_mut(), flat.as_ptr(), n, rnd.as_ptr(), rec.as_mut_ptr(), ffi::TECDSA_HOST) })?;
        Ok(rec)
    }

    /// The sampling half of `MessageA::a`, `MessageB::b`, `AliceProof::generate`, `PDLwSlackProof::prove` and `SignKeys::create`
    /// for a batch of sessions, drawn on the device from one 32-byte seed (`tecdsa_gg20_sample_randomness`): the `rnd` that
    /// `offline_records` takes and one status byte per unit (0, or `TECDSA_ST_SAMPLING`).  Unit `2 s + position` has element id
    /// `first_unit + 2 s + position`; a (seed, element id) pair must NEVER be used twice — a fresh seed from the OS CSPRNG per
    /// call, or one seed with disjoint `first_unit` ranges.
    pub fn sample_randomness(e: &Engine, ks: &KeySets, sessions: &[[u32; 3]], seed: &[u8; 32], first_unit: u64) -> Result<(Vec<u32>, Vec<u8>), EngineError> {
        let n = sessions.len();
        let flat: Vec<u32> = sessions.iter().flat_map(|s| s.iter().copied()).collect();
        let mut words = [0u32; 8];
        for (w, c) in words.iter_mut().zip(seed.chunks_exact(4)) {
            *w = u32::from_le_bytes([c[0], c[1], c[2], c[3]]);
        }
        let mut rnd = vec![0u32; 2 * n * ffi::TECDSA_RND_LIMBS];
        let mut status = vec![0u8; 2 * n];
        let rc = unsafe { ffi::tecdsa_gg20_sample_randomness(e.raw(), ks.raw(), flat.as_ptr(), n, words.as_ptr(), first_unit, rnd.as_mut_ptr(), status.as_mut_ptr(), ffi::TECDSA_HOST) };
        words = [0u32; 8];
        let _ = words;
        check(rc)?;
        Ok((rnd, status))
    }

    /// `party_two::PartialSig::compute` for a batch (two_party_ecdsa/lindell_2017/party_two.rs:390-424) with `rho` (< q^2) and the
    /// randomness of `Paillier::encrypt` explicit: c3 per element, or `None` where the reference would panic (k2 = 0).
    /// `n[key_idx[i]]` is the Paillier modulus of element i.
    #[allow(clippy::too_many_arguments)]
    pub fn l17_partial_sig(e: &Engine, n: &[BigInt], key_idx: &[u32], c_key: &[BigInt], x2: &[Scalar<Secp256k1>], k2: &[Scalar<Secp256k1>],
                           eph_other_public: &[Point<Secp256k1>], message: &[BigInt], rho: &[BigInt], randomness: &[BigInt]) -> Result<Vec<Option<BigInt>>, EngineError> {
        let cnt = c_key.len();
        let pack = |v: &[BigInt], limbs: usize| -> Vec<u32> { v.iter().flat_map(|x| to_limbs(x, limbs)).collect() };
        let q = Scalar::<Secp256k1>::group_order();
        let msg: Vec<BigInt> = message.iter().map(|m| m.mod_floor(q)).collect();
        let (nl, ck, ml, rl, rr) = (pack(n, 64), pack(c_key, 128), pack(&msg, 8), pack(rho, 16), pack(randomness, 64));
        let x2l: Vec<u32> = x2.iter().flat_map(scalar_to_limbs).collect();
        let k2l: Vec<u32> = k2.iter().flat_map(scalar_to_limbs).collect();
        let pl: Vec<u32> = eph_other_public.iter().flat_map(point_to_limbs).collect();
        let (mut c3, mut st) = (vec![0u32; cnt * 128], vec![255u8; cnt]);
        check(unsafe {
            ffi::tecdsa_l17_partial_sig_batch(e.raw(), nl.as_ptr(), key_idx.as_ptr(), n.len(), ck.as_ptr(), x2l.as_ptr(), k2l.as_ptr(), pl.as_ptr(), ml.as_ptr(),
                                              rl.as_ptr(), rr.as_ptr(), c3.as_mut_ptr(), st.as_mut_ptr(), cnt, ffi::TECDSA_HOST)
        })?;
        Ok((0..cnt).map(|i| if st[i] == 0 { Some(from_limbs(&c3[i * 128..(i + 1) * 128])) } else { None }).collect())
    }

    /// `party_one::Signature::compute_with_recid` for a batch (party_one.rs:519-564) under Paillier key rows of an uploaded key set:
    /// (r, s, recid) per element, or `None` where the reference would panic (k1 = 0).
    pub fn l17_sign(e: &Engine, ks: &KeySets, key_row: &[u32], c3: &[BigInt], k1: &[Scalar<Secp256k1>], eph_other_public: &[Point<Secp256k1>])
                    -> Result<Vec<Option<(BigInt, BigInt, u8)>>, EngineError> {
        let cnt = c3.len();
        let cl: Vec<u32> = c3.iter().flat_map(|x| to_limbs(x, 128)).collect();
        let kl: Vec<u32> = k1.iter().flat_map(scalar_to_limbs).collect();
        let pl: Vec<u32> = eph_other_public.iter().flat_map(point_to_limbs).collect();
        let (mut r, mut s, mut rec, mut st) = (vec![0u32; cnt * 8], vec![0u32; cnt * 8], vec![0u8; cnt], vec![255u8; cnt]);
        check(unsafe {
            ffi::tecdsa_l17_sign_batch(e.raw(), ks.raw(), key_row.as_ptr(), cl.as_ptr(), kl.as_ptr(), pl.as_ptr(), r.as_mut_ptr(), s.as_mut_ptr(), rec.as_mut_ptr(),
                                       st.as_mut_ptr(), cnt, ffi::TECDSA_HOST)
        })?;
        Ok((0..cnt).map(|i| if st[i] == 0 { Some((from_limbs(&r[i * 8..(i + 1) * 8]), from_limbs(&s[i * 8..(i + 1) * 8]), rec[i])) } else { None }).collect())
    }
}
