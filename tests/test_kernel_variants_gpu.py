"""Every compiled shape of the N-adic job kernels, the Kaliski fallback of the offline stage's inverses modulo N^2 and the
unsplit offline driver, each compared with the oracle and bit for bit with the default configuration; the non-invertible
ciphertext path of the offline stage (nadic_inv_kernel with ok = 0); and lane groups of one warp that leave the Kaliski loop
of group_modinv after very different numbers of steps.

The kernel shape is chosen by environment variables that the library reads once per process (csrc/capi.cu nadic_shape(),
tecdsa_hensel_inverse(); csrc/gg20.cu split_min_sessions()), so each configuration runs in a fresh interpreter, one after
the other.  The parent builds the inputs and the oracle's expectations once; the child runs the GPU payload and writes its
outputs and the names of the kernels it launched to an .npz file.  An unrecognised TECDSA_NADIC_SHAPE is ignored by the
library, so every configuration also asserts, from the per-launch profile, which instantiation actually ran."""
import os
import pickle
import random
import subprocess
import sys

import numpy as np
import pytest

from oracle import gg20_oracle as o
from oracle.sampling import Drbg, sample_unit

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
VARIANT_ENV = ("TECDSA_NADIC_SHAPE", "TECDSA_HENSEL", "TECDSA_SPLIT")
NADIC_INV, KALISKI_4096 = "nadic_inv_kernel<64,8>", "inv_jobs_kernel<128,8>"
# id -> (environment, N-adic instantiation modulo N^2, N-adic instantiation modulo p^2 / q^2)
CONFIGS = {
    "default": ({}, "nadic_jobs_kernel<64,8,4>", "nadic_jobs_kernel<32,4,4>"),
    "nn-8-1": ({"TECDSA_NADIC_SHAPE": "8,1"}, "nadic_jobs_kernel<64,8,1>", "nadic_jobs_kernel<32,4,4>"),
    "nn-4-3": ({"TECDSA_NADIC_SHAPE": "4,3"}, "nadic_jobs_kernel<64,4,3>", "nadic_jobs_kernel<32,4,4>"),
    "nn-4-1": ({"TECDSA_NADIC_SHAPE": "4,1"}, "nadic_jobs_kernel<64,4,1>", "nadic_jobs_kernel<32,4,4>"),
    "pp-4-1": ({"TECDSA_NADIC_SHAPE": "8,4,4,1"}, "nadic_jobs_kernel<64,8,4>", "nadic_jobs_kernel<32,4,1>"),
    "pp-2-1": ({"TECDSA_NADIC_SHAPE": "8,4,2,1"}, "nadic_jobs_kernel<64,8,4>", "nadic_jobs_kernel<32,2,1>"),
    "kaliski": ({"TECDSA_HENSEL": "0"}, "nadic_jobs_kernel<64,8,4>", "nadic_jobs_kernel<32,4,4>"),
    "nosplit": ({"TECDSA_SPLIT": "0"}, "nadic_jobs_kernel<64,8,4>", "nadic_jobs_kernel<32,4,4>"),
}
BIG_SESSIONS = 2049                 # above the 2048-session split threshold of csrc/gg20.cu, odd: unequal halves
CHILD_TIMEOUT_S = 900


# ------------------------------------------------------------------------------------------------ shared inputs
def _inverse_session_inputs(keyset):
    """Five two-signer sessions (10 units) over one key set with three units whose ciphertexts are not units modulo N^2.
    TPI_NADIC_INV = 8 puts 4 units in one warp of nadic_inv_kernel, so the broken units 1, 2 and 5 share warps with healthy
    ones:
      unit 1: r_k = p of its own key  -> MessageA.c = 0 mod p: the peer (unit 0) cannot invert it in AliceProof::verify;
      unit 2: r_k = 0                 -> MessageA.c = 0: the peer (unit 3) rejects likewise;
      unit 5: r_gamma = p of the peer's key -> the MtA response to unit 4 is 0 mod p: unit 4's decryption of it gives
              a share that fails verify_proofs_get_alpha."""
    pairs = [(0, 1), (1, 2), (2, 0), (0, 2), (2, 1)]
    rng = Drbg(0xB2000B, "offline-inverse")
    sess, rnds, oracle_in = [], [], []
    for a, b in pairs:
        s_l, keys = [a + 1, b + 1], [keyset[a], keyset[b]]
        r = [sample_unit(rng, keys, s_l, p) for p in range(2)]
        sess.append((0, a, b)); rnds += r; oracle_in.append((keys, s_l, r))
    rnds[1].r_k = keyset[pairs[0][1]].dk.p
    rnds[2].r_k = 0
    rnds[5].r_gamma = keyset[pairs[2][0]].dk.p
    return sess, rnds, oracle_in


@pytest.fixture(scope="module")
def inverse_case(keyset):
    """(sessions, randomness, per-session oracle results) of _inverse_session_inputs, computed once"""
    sess, rnds, oracle_in = _inverse_session_inputs(keyset)
    return sess, rnds, [o.offline_session(*x) for x in oracle_in]


def _edge_inputs():
    """test_l012_gpu.test_paillier_nadic_edge_cases' odd moduli and operands, 101 of them (neither a multiple of the 8 nor of
    the 4 groups per warp)"""
    rng = random.Random(0x7A1)
    B = 2048
    ns = [3, (1 << B) - 1, rng.getrandbits(1500) | 1, rng.getrandbits(B - 1) | 1 | (1 << (B - 2)), (1 << (B - 1)) + 1, 5 ** 800]
    ns += [rng.getrandbits(B) | 1 | (1 << (B - 1)) for _ in range(10)]
    n = 101
    idx = [i % len(ns) for i in range(n)]
    c = [rng.getrandbits(4096) for _ in range(n)]
    k = [rng.getrandbits(2048) for _ in range(n)]
    c[0] = 0; c[1] = 1; k[2] = 0; k[3] = 1; c[4] = (1 << 4096) - 1; k[5] = (1 << 2048) - 1
    for j in range(6, 22):
        c[j] = ns[idx[j]] ** 2 - 1 - (j & 1) * rng.getrandbits(40)
    c2 = [rng.getrandbits(4096) for _ in range(n)]
    m = [rng.getrandbits(2048) for _ in range(n)]
    r = [rng.getrandbits(2048) for _ in range(n)]
    return ns, idx, c, k, c2, m, r


def _decrypt_inputs(keyset):
    """37 ciphertexts that are units modulo N^2 (for other values the reference's L() divides a negative number, and truncated
    and floor division disagree): random ones, 1, N^2 - 1, and c + j N^2 up to the full 4096-bit operand width, which reaches
    the top chunk of the p-adic lift"""
    from math import gcd
    rng = random.Random(0xDEC)
    idx, cs = [], []
    for i in range(37):
        row = i % 3
        N = keyset[row].dk.p * keyset[row].dk.q
        NN = N * N
        while True:
            c = rng.randrange(2, NN)
            if gcd(c, N) == 1:
                break
        kind = i // 3 % 4
        if kind == 1:
            c = 1 if i % 2 else NN - 1
        elif kind == 2:
            c += ((1 << 4096) - 1 - c) // NN * NN         # the largest c + j N^2 below 2^4096
        idx.append(row); cs.append(c)
    return idx, cs


def _proof_inputs(keyset):
    """AliceProof, BobProofExt and PDLwSlackProof batches made by the oracle, each with one tampered proof"""
    rng = Drbg(0xB2000C, "variant-proofs")
    q3 = o.Q ** 3
    eks, sts = keyset[0].paillier_key_vec, keyset[0].h1_h2_n_tilde_vec
    n = 13
    a_er, a_sr = [i % 3 for i in range(n)], [(i // 3) % 3 for i in range(n)]
    alice = {k: [] for k in ("a", "c", "r", "al", "be", "ga", "ro")}
    for i in range(n):
        ek, st = eks[a_er[i]], sts[a_sr[i]]
        a, r = rng.scalar(), rng.unit_mod(ek.n)
        for k, v in zip(alice, (a, o.paillier_encrypt(ek, a, r), r, rng.below(q3), rng.unit_mod(ek.n), rng.below(q3 * st.N), rng.below(o.Q * st.N))):
            alice[k].append(v)
    alice_bad = list(alice["c"]); alice_bad[4] += 1
    nb = 9
    b_er, b_sr = [i % 3 for i in range(nb)], [(i + 2) % 3 for i in range(nb)]
    bob = {k: [] for k in ("a_enc", "mta", "X", "t", "z", "e", "s", "s1", "s2", "t1", "t2", "u")}
    for i in range(nb):
        ek, st = eks[b_er[i]], sts[b_sr[i]]
        a, b = rng.scalar(), rng.scalar()
        enc_a = o.paillier_encrypt(ek, a, rng.unit_mod(ek.n))
        bp, r = rng.below(ek.n), rng.unit_mod(ek.n)
        mta = o.paillier_add(ek, o.paillier_mul(ek, enc_a, b), o.paillier_encrypt(ek, bp, r))
        w, u = o.bob_proof_generate(enc_a, mta, b, bp, ek, st, r, True, rng.below(q3), rng.unit_mod(ek.n), rng.below(o.Q ** 2 * ek.n),
                                    rng.below(o.Q * st.N), rng.below(q3 * st.N), rng.below(o.Q * st.N), rng.below(q3 * st.N))
        for k, v in (("a_enc", enc_a), ("mta", mta), ("X", o.pt_mul(o.G, b)), ("u", u), *((f, getattr(w, f)) for f in ("t", "z", "e", "s", "s1", "s2", "t1", "t2"))):
            bob[k].append(v)
    bob["t1"][7] += 1
    npd = 9
    p_er, p_sr = [i % 3 for i in range(npd)], [(i + 1) % 3 for i in range(npd)]
    pdl = {k: [] for k in ("c", "Q", "G", "z", "u1", "u2", "u3", "s1", "s2", "s3")}
    for i in range(npd):
        ek, st = eks[p_er[i]], sts[p_sr[i]]
        x, r = rng.scalar(), rng.unit_mod(ek.n)
        c = o.paillier_encrypt(ek, x, r)
        Gp = o.pt_mul(o.G, rng.scalar()); Qp = o.pt_mul(Gp, x)
        w = o.pdl_prove(x, r, c, ek, Qp, Gp, st.g, st.ni, st.N, rng.below(q3), 1 + rng.below(ek.n - 2), rng.below(o.Q * st.N), rng.below(q3 * st.N))
        for k, v in (("c", c), ("Q", Qp), ("G", Gp), *((f, getattr(w, f)) for f in ("z", "u1", "u2", "u3", "s1", "s2", "s3"))):
            pdl[k].append(v)
    pdl["z"][5] = 0                                   # not invertible modulo N_tilde: the reference's unwrap() site
    return dict(alice=(a_er, a_sr, alice, alice_bad), bob=(b_er, b_sr, bob), pdl=(p_er, p_sr, pdl))


# ------------------------------------------------------------------------------------------------ child process
def _child_main(inp_path, out_path, big):
    """Runs in a fresh interpreter with the configuration's environment: the GPU payload, outputs to out_path (.npz)."""
    import __graft_entry__ as entry
    pkg = entry.load_package()
    from mpecdsa_b200 import gg20
    from tests.golden import fixtures
    with open(inp_path, "rb") as f:
        I = pickle.load(f)
    L = pkg.ints_to_limbs
    eng = pkg.Engine(0)
    keysets = fixtures.load_all_keysets()
    ks1, ks8 = gg20.KeySets(eng, keysets[:1]), gg20.KeySets(eng, keysets)
    out = {}
    ns, idx, c, k, c2, m, r = I["edge"]
    out["paillier_mul"] = L(eng.paillier_mul(ns, idx, c, k, k_limbs=64), 128)
    out["paillier_add"] = L(eng.paillier_add(ns, idx, c, c2), 128)
    out["paillier_encrypt"] = L(eng.paillier_encrypt(ns, idx, m, r), 128)
    didx, dcs = I["decrypt"]
    out["paillier_decrypt"] = L(eng.paillier_decrypt(ks1.handle, didx, dcs), 64)
    er, sr, al, al_bad = I["alice"]
    pf = gg20.alice_proof_generate(eng, ks1, er, sr, al["a"], al["c"], al["r"], al["al"], al["be"], al["ga"], al["ro"])
    for f, width in (("z", 64), ("e", 8), ("s", 64), ("s1", 28), ("s2", 92)):
        out["alice_" + f] = L(pf[f], width)
    out["alice_status"] = gg20.alice_proof_verify(eng, ks1, er, sr, al_bad, pf["z"], pf["e"], pf["s"], pf["s1"], pf["s2"])
    er, sr, bob = I["bob"]
    out["bob_status"] = gg20.bob_proof_verify(eng, ks1, er, sr, bob["a_enc"], bob["mta"], bob, bob["X"], bob["u"])
    er, sr, pd = I["pdl"]
    out["pdl_status"] = gg20.pdl_verify(eng, ks1, er, sr, pd["c"], pd["Q"], pd["G"], *(pd[f] for f in ("z", "u1", "u2", "u3", "s1", "s2", "s3")))
    off_sess, off_rnd = I["offline"]
    res = gg20.offline_batch(eng, ks1, off_sess, off_rnd)
    for f in ("status", "R", "sigma", "t_vec", "digest"):
        out["offline_" + f] = getattr(res, f)
    sess, rnd = I["records"]
    rec = np.zeros((1, 2 * len(sess), pkg.REC_BYTES), dtype=np.uint8)
    eng.offline_records(ks8, None, sess, len(sess), rnd, rec, pkg.HOST)
    out["records"] = rec[0]
    # which kernels ran: the per-launch profile of one offline call and one decryption
    out["prof_offline"] = np.array(sorted(eng.profile_step(lambda: gg20.offline_batch(eng, ks1, off_sess, off_rnd))))
    out["prof_decrypt"] = np.array(sorted(eng.profile_step(lambda: eng.paillier_decrypt(ks1.handle, didx, dcs))))
    if big:
        sess, rnd = I["big"]
        l0 = eng.launch_count()
        res = gg20.offline_batch(eng, ks8, sess, rnd)
        out["big_launches"] = np.array(eng.launch_count() - l0)
        for f in ("status", "R", "sigma", "t_vec", "digest"):
            out["big_" + f] = getattr(res, f)
    ks1.free(); ks8.free()
    eng.close()
    np.savez(out_path, **out)


# ------------------------------------------------------------------------------------------------ parent side
@pytest.fixture(scope="module")
def variant_inputs(tmp_path_factory, keyset, inverse_case):
    """The inputs every child runs (pickled once) and what the oracle and the C twin say about them."""
    from mpecdsa_b200 import gg20
    from oracle import twin
    from tests.golden import fixtures
    keysets = fixtures.load_all_keysets()
    sess, rnds, off_want = inverse_case
    I = dict(edge=_edge_inputs(), decrypt=_decrypt_inputs(keyset), offline=(sess, gg20.pack_randomness(rnds)),
             records=gg20.synthetic_batch(keysets, 48, 0xB2000D), big=gg20.synthetic_batch(keysets[:2], BIG_SESSIONS, 11), **_proof_inputs(keyset))
    path = tmp_path_factory.mktemp("variants") / "inputs.pkl"
    with open(path, "wb") as f:
        pickle.dump(I, f)
    ns, idx, c, k, c2, m, r = I["edge"]
    want = dict(
        paillier_mul=[pow(cc, kk, ns[i] ** 2) for i, cc, kk in zip(idx, c, k)],
        paillier_add=[x * y % ns[i] ** 2 for i, x, y in zip(idx, c, c2)],
        paillier_encrypt=[(1 + mm * ns[i]) * pow(rr, ns[i], ns[i] ** 2) % ns[i] ** 2 for i, mm, rr in zip(idx, m, r)],
        paillier_decrypt=[o.paillier_decrypt(keyset[i].dk, x) for i, x in zip(*I["decrypt"])])
    er, sr, al, al_bad = I["alice"]
    eks, sts = keyset[0].paillier_key_vec, keyset[0].h1_h2_n_tilde_vec
    want["alice"] = [o.alice_proof_generate(al["a"][i], al["c"][i], eks[er[i]], sts[sr[i]], al["r"][i], al["al"][i], al["be"][i], al["ga"][i], al["ro"][i])
                     for i in range(len(er))]
    want["alice_ok"] = [o.alice_proof_verify(pf, cc, eks[e], sts[s]) for pf, cc, e, s in zip(want["alice"], al_bad, er, sr)]
    er, sr, bob = I["bob"]
    want["bob_ok"] = [o.bob_proof_ext_verify(o.BobProof(*(bob[f][i] for f in ("t", "z", "e", "s", "s1", "s2", "t1", "t2"))), bob["u"][i], bob["a_enc"][i],
                                             bob["mta"][i], eks[er[i]], sts[sr[i]], bob["X"][i]) for i in range(len(er))]
    er, sr, pd = I["pdl"]
    want["pdl_ok"] = [o.pdl_verify(o.PDLwSlackProof(*(pd[f][i] for f in ("z", "u1", "u2", "u3", "s1", "s2", "s3"))), pd["c"][i], eks[er[i]], pd["Q"][i],
                                   pd["G"][i], sts[sr[i]].g, sts[sr[i]].ni, sts[sr[i]].N) for i in range(len(er))]
    assert want["alice_ok"].count(False) == 1 and want["bob_ok"].count(False) == 1 and want["pdl_ok"].count(False) == 1
    want["offline"] = off_want
    want["records"] = twin.offline_batch(twin.KeyTables(keysets), *I["records"], 8)
    return path, want


_RUNS = {}


def _run_config(name, inp_path, out_dir):
    """Start one child for configuration `name` (cached: the default run is the reference of every other one)."""
    if name in _RUNS:
        return _RUNS[name]
    env = {k: v for k, v in os.environ.items() if k not in VARIANT_ENV}     # TECDSA_B200_LIB, CUDA_VISIBLE_DEVICES are inherited
    env.update(CONFIGS[name][0])
    out_path = os.path.join(str(out_dir), f"{name}.npz")
    big = name in ("default", "nosplit")
    code = f"import sys; sys.path.insert(0, {ROOT!r}); from tests.test_kernel_variants_gpu import _child_main; _child_main({str(inp_path)!r}, {out_path!r}, {big})"
    flags = ["-s"] if sys.flags.no_user_site else []
    p = subprocess.run([sys.executable, *flags, "-c", code], cwd=ROOT, env=env, timeout=CHILD_TIMEOUT_S, capture_output=True, text=True)
    assert p.returncode == 0, f"{name}: child failed (rc={p.returncode})\n{p.stdout[-4000:]}\n{p.stderr[-4000:]}"
    with np.load(out_path) as z:
        _RUNS[name] = {k: z[k] for k in z.files}
    return _RUNS[name]


def _be(limbs):
    return np.ascontiguousarray(limbs[:, ::-1]).astype(">u4").view(np.uint8).reshape(limbs.shape[0], 32)


@pytest.mark.parametrize("name", list(CONFIGS))
def test_kernel_variant_matches_oracle_and_default(name, variant_inputs, tmp_path_factory, pkg):
    from mpecdsa_b200 import gg20
    inp_path, want = variant_inputs
    out_dir = tmp_path_factory.mktemp(f"variant-{name}")
    got = _run_config(name, inp_path, out_dir)
    ref = _run_config("default", inp_path, tmp_path_factory.mktemp("variant-default-ref"))
    ints = pkg.limbs_to_ints
    # the instantiations that ran
    _, n64, n32 = CONFIGS[name]
    prof_off, prof_dec = set(got["prof_offline"].tolist()), set(got["prof_decrypt"].tolist())
    assert {k for k in prof_off if k.startswith("nadic_jobs_kernel")} == {n64, n32}, prof_off
    assert {k for k in prof_dec if k.startswith("nadic_jobs_kernel")} == {n32}, prof_dec
    if name == "kaliski":
        assert KALISKI_4096 in prof_off and NADIC_INV not in prof_off, prof_off
    else:
        assert NADIC_INV in prof_off and KALISKI_4096 not in prof_off, prof_off
    # values against the oracle
    for f in ("paillier_mul", "paillier_add", "paillier_encrypt", "paillier_decrypt"):
        assert ints(got[f]) == want[f], (name, f)
    for f in ("z", "e", "s", "s1", "s2"):
        assert ints(got["alice_" + f]) == [getattr(pf, f) for pf in want["alice"]], (name, f)
    assert [s == 0 for s in got["alice_status"]] == want["alice_ok"] and got["alice_status"][4] == pkg.ST_HASH_MISMATCH
    assert [s == 0 for s in got["bob_status"]] == want["bob_ok"] and got["bob_status"][7] == pkg.ST_HASH_MISMATCH
    assert [s == 0 for s in got["pdl_status"]] == want["pdl_ok"] and got["pdl_status"][5] == pkg.ST_PDL_VERIFY
    _assert_offline_matches_oracle(pkg, gg20, got, want["offline"])
    tw, rec = want["records"], got["records"]
    assert not tw.status.any() and not rec[:, 0].any()
    assert np.array_equal(rec[:, 164:196], _be(tw.digest)) and np.array_equal(rec[:, 34:66], _be(tw.sigma)) and np.array_equal(rec[:, 66:98], _be(tw.k))
    assert np.array_equal(rec[:, 2:34], _be(tw.R[:, :8])) and np.array_equal(rec[:, 1], 2 + (tw.R[:, 8] & 1).astype(np.uint8))
    assert np.array_equal(rec[:, 99:131], _be(tw.t_vec[:, :8])) and np.array_equal(rec[:, 132:164], _be(tw.t_vec[:, 16:24]))
    assert np.array_equal(rec[:, 98], 2 + (tw.t_vec[:, 8] & 1).astype(np.uint8)) and not rec[:, 196:].any()
    # and bit for bit with the default configuration
    for f in got:
        if not f.startswith(("prof_", "big_launches")):
            assert np.array_equal(got[f], ref[f]), (name, f)
    if name == "nosplit":
        assert not got["big_status"].any()
        # split (default): both halves run the whole launch sequence on child contexts and their counts are added to the
        # caller's context (tecdsa_internal_offline); unsplit: one sequence on the caller's context
        assert int(ref["big_launches"]) > int(got["big_launches"]) > 0, (int(ref["big_launches"]), int(got["big_launches"]))


def _assert_offline_matches_oracle(pkg, gg20, got, want_sessions):
    """A unit the oracle rejects has the oracle's status.  The oracle, like the reference, stops a session at the first round
    in which a party rejects, so its peer keeps status 0 without outputs; the batch runs every round for every unit and the
    peer then fails a later check of its own on messages the reference never sends, so on the device the peer's status is
    non-zero.  Sessions the oracle completes are bit-equal to it."""
    status = got["offline_status"]
    for s, ws in enumerate(want_sessions):
        if any(w.status for w in ws):
            for p in range(2):
                assert status[2 * s + p] == ws[p].status if ws[p].status else status[2 * s + p] != 0, (s, p, list(status))
            continue
        assert not status[2 * s:2 * s + 2].any(), (s, list(status))
        for p in range(2):
            u = 2 * s + p
            assert gg20.unpack_point(pkg.limbs_to_ints(got["offline_R"][u:u + 1])[0]) == ws[p].R
            assert pkg.limbs_to_ints(got["offline_sigma"][u:u + 1])[0] == ws[p].sigma_i
            assert [gg20.unpack_point(v) for v in pkg.limbs_to_ints(got["offline_t_vec"][u].reshape(2, 16))] == ws[p].t_vec
            assert int.from_bytes(got["offline_digest"][u].tobytes(), "little").to_bytes(32, "big") == ws[p].transcript


# ------------------------------------------------------------------------------------------------ B: offline stage, in process
def test_offline_noninvertible_ciphertexts(engine, pkg, keyset, inverse_case):
    """Ciphertexts that are not units modulo N^2, next to healthy units in the same warps of nadic_inv_kernel: every unit
    the oracle rejects has the oracle's status, its peer is not reported OK, and the healthy sessions' R, sigma_i, t_vec and
    transcript digest are bit-equal to the oracle.
    The status alone cannot tell a wrong `ok` flag from a right one (the reference maps every failed proof check to
    InvalidKey, and a wrong inverse also fails the challenge check); what this pins is agreement with the oracle on the
    failing units and that their neighbours in the warp are unaffected.  The Kaliski fallback (TECDSA_HENSEL=0) runs the same
    inputs in test_kernel_variant_matches_oracle_and_default[kaliski]."""
    from mpecdsa_b200 import gg20
    sess, rnds, want = inverse_case
    ks = gg20.KeySets(engine, [keyset])
    res = gg20.offline_batch(engine, ks, sess, gg20.pack_randomness(rnds))
    ks.free()
    got = {"offline_" + f: getattr(res, f) for f in ("status", "R", "sigma", "t_vec", "digest")}
    assert [w.status for w in want[0] + want[1] + want[2]] == [pkg.ST_INVALID_KEY, 0, 0, pkg.ST_INVALID_KEY, pkg.ST_INVALID_KEY, 0]
    _assert_offline_matches_oracle(pkg, gg20, got, want)


# ------------------------------------------------------------------------------------------------ C: Kaliski divergence
def _fib_pair(bits):
    """the largest consecutive Fibonacci numbers (a, n) with n odd and below 2^bits: the longest inversion for their size"""
    a, b, best = 1, 2, None
    while b < 1 << bits:
        if b & 1:
            best = (a, b)
        a, b = b, a + b
    return best


def _modinv_operands(bits, count, moduli, primes, rng):
    """(a, index into moduli) for `count` operands: odd slots are slow (a Fibonacci ratio, or random full width), even slots
    fast (1, 2, 2^j, n - 1), degenerate (n, 0, >= n, k*n + 1) or a multiple of a 1024-bit prime factor of moduli[0]"""
    fast = [lambda n: 1, lambda n: 2, lambda n: 1 << rng.randrange(3, bits - 1), lambda n: n - 1]
    edge = [lambda n: n, lambda n: 0, lambda n: n + 1 + rng.getrandbits(bits - 8), lambda n: rng.randrange(1, 4) * n + 1]
    out = []
    for i in range(count):
        j = i % len(moduli)
        if i % 2:
            j = 1 if i % 4 == 1 else 2
            a = _fib_pair(bits)[0] if j == 1 else rng.getrandbits(bits)
        elif i % 6 == 2:
            j = 3                                                   # the short modulus: n + x and 3n + 1 stay below 2^bits
            a = edge[(i // 6) % len(edge)](moduli[j])
        elif i % 6 == 4:
            j = 0
            f = primes[(i // 6) % len(primes)]
            a = f * rng.randrange(2, moduli[0] // f)                # gcd(a, n) >= f
        else:
            a = fast[(i // 6) % len(fast)](moduli[j])
        assert 0 <= a < 1 << bits
        out.append((a, j))
    return out


@pytest.mark.parametrize("bits", [2048, 4096])
def test_modinv_divergent_groups_in_one_warp(engine, pkg, bits):
    """Every warp of inv_jobs_kernel (8 groups at 2048 bits, 4 at 4096) mixes inversions that finish in a few steps (1, 2,
    2^j, n-1, 0, n) with ones that take the longest (consecutive Fibonacci numbers, random full-width operands): the
    branch-free tail of group_modinv must use each group's own step count.  Also operands >= n, k*n + 1, and multiples of
    a 1024-bit prime factor of n = p*q (a large gcd).  Once with one modulus per operand and once through the mod_idx
    gather."""
    from tests.golden import fixtures
    ks = fixtures.load_keyset(0)
    rng = random.Random(bits * 3 + 1)
    primes = [ks[0].dk.p, ks[0].dk.q] if bits == 2048 else [ks[0].dk.p, ks[0].dk.q, ks[1].dk.p, ks[1].dk.q]
    pq = 1
    for f in primes:
        pq *= f
    moduli = [pq, _fib_pair(bits)[1], rng.getrandbits(bits) | 1 | (1 << (bits - 1)), rng.getrandbits(bits - 3) | 1 | (1 << (bits - 4))]
    K = bits // 32
    count = 8 * (12 if bits == 2048 else 6) + 3
    ops = _modinv_operands(bits, count, moduli, primes, rng)
    a = [x for x, _ in ops]
    mods = [moduli[j] for _, j in ops]

    def want(x, n):
        try:
            return pow(x, -1, n)
        except ValueError:
            return None

    expect = [want(x, n) for x, n in zip(a, mods)]
    assert expect.count(None) >= 4 and sum(1 for e in expect if e is not None) >= count // 2
    assert engine.mod_inv(a, mods, bits) == expect
    # the same operands through the modulus index
    pkg._bind_l01(engine.lib)
    A, M = pkg.ints_to_limbs(a, K), pkg.ints_to_limbs(moduli, K)
    idx = np.array([j for _, j in ops], dtype=np.uint32)
    out, ok = np.zeros_like(A), np.zeros(count, dtype=np.uint8)
    engine._ck(engine.lib.tecdsa_modinv_batch(engine._ctx, bits, A.ctypes.data, M.ctypes.data, idx.ctypes.data, len(moduli), out.ctypes.data,
                                              ok.ctypes.data, count, pkg.HOST), "modinv_batch")
    assert [v if f else None for v, f in zip(pkg.limbs_to_ints(out), ok)] == expect
