"""Carry-stress tests of the lane-group big-integer kernels: every output compared with Python integers (or GMP), on the
structured operands of tests/carry_operands.py instead of uniform random limbs.  Those operands reach the carry lookahead
across all-ones lanes (group_carry's propagate path, the second carry word of mont_mul / rows_finish), the all-ones start
of the N-adic product's second pass, the block sums of mont_sqr, all-ones and boundary exponent windows, short exponent
widths, and the chunked launch loop of tecdsa_modexp_batch.  tests/test_carry_operands.py shows on the CPU that the
families reach those paths.

Batch sizes are never multiples of the groups per warp, so groups with different operands (and moduli) share warps."""
import os
import pickle
import random
import subprocess
import sys
from math import gcd

import numpy as np
import pytest

from tests import carry_operands as co

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODEXP_TPIS = {1024: (4, 8, 16), 2048: (4, 8, 16, 32), 4096: (8, 16, 32)}
JOB_TPI = {2048: 4, 4096: 8}                  # exp_jobs_kernel / inv_jobs_kernel lanes per operand (modmul, modinv)


def _union_moduli(bits, tpis, rng):
    out = []
    for t in tpis:
        out += [n for n in co.moduli(bits, t, rng) if n not in out]
    return out


def _union_structured(bits, tpis, rng):
    out = []
    for t in tpis:
        out += co.structured(bits, t, rng)
    return out


# ------------------------------------------------------------------------------------------------ 1. modexp, every shape
@pytest.mark.parametrize("bits", [1024, 2048, 4096])
def test_modexp_structured_every_tpi_and_squaring(engine, bits):
    """tecdsa_modexp_batch on structured moduli, bases and exponents at every TPI set_tpi accepts for the width, with the
    squaring through mont_mul and through mont_sqr; exponents of 1, 2, 3 and 65 limbs (all-ones windows, 2^j and 2^j - 1 on
    window and limb boundaries, runs)."""
    rng = random.Random(0xCA77 + bits)
    tpis = MODEXP_TPIS[bits]
    ms = _union_moduli(bits, tpis, rng)
    bases = _union_structured(bits, tpis, rng)
    for n in ms:
        bases += co.residues(n, bits)
    cases = []
    for el, count in ((1, 101), (2, 67), (3, 101), (65, 37 if bits == 4096 else 45)):
        es = co.exponents(32 * el, rng)
        b = [bases[(7 * i + el) % len(bases)] for i in range(count)]
        e = [es[i % len(es)] for i in range(count)]
        m = [ms[(3 * i + el) % len(ms)] for i in range(count)]
        cases.append((el, b, e, m, [pow(x, y, z) for x, y, z in zip(b, e, m)]))
    try:
        for tpi in tpis:
            engine.set_tpi(bits, tpi)
            for sqr in (0, 1):
                engine.set_option("sqr", sqr)
                for el, b, e, m, want in cases:
                    got, st = engine.mod_pow(b, e, m, mod_bits=bits, exp_bits=32 * el)
                    assert not st.any(), (bits, tpi, sqr, el)
                    bad = [i for i in range(len(want)) if got[i] != want[i]]
                    assert not bad, (bits, tpi, sqr, el, bad[:8])
    finally:
        engine.set_option("sqr", 0)
        for w in (1024, 2048, 4096):
            engine.set_tpi(w, 0)


# ------------------------------------------------------------------------------------------------ 2. modmul
@pytest.mark.parametrize("bits", [2048, 4096])
def test_modmul_structured(engine, bits):
    """tecdsa_modmul_batch over the modulus families x boundary residues, lane-aligned operands, and pairs whose product is
    0, 1 or n - 1 modulo n"""
    rng = random.Random(0x33 + bits)
    tpi = JOB_TPI[bits]
    ms = co.moduli(bits, tpi, rng)
    lv = co.structured(bits, tpi, rng)
    a, b, m = [], [], []
    for n in ms:
        rs = co.residues(n, bits)
        pairs = co.product_pairs(n, rng) + [(x, y) for x in rs for y in rs[:3]]
        pairs += [(lv[(5 * k + len(a)) % len(lv)], lv[(3 * k + 1) % len(lv)]) for k in range(12)]
        for x, y in pairs:
            a.append(x); b.append(y); m.append(n)
    if len(a) % (32 // tpi) == 0:
        a.append(1); b.append(1); m.append(ms[0])
    got = engine.mod_mul(a, b, m, bits)
    bad = [i for i in range(len(a)) if got[i] != a[i] * b[i] % m[i]]
    assert not bad, [(hex(a[i])[:20], hex(b[i])[:20], hex(m[i])[:20]) for i in bad[:4]]


# ------------------------------------------------------------------------------------------------ 3. modinv
@pytest.mark.parametrize("bits", [2048, 4096])
def test_modinv_structured(engine, bits):
    """tecdsa_modinv_batch (inv_jobs_kernel<64,4> / <128,8>): a = 2^j across lane boundaries, n-1, n-2, a >= n (R-1, n+1),
    a = n and 2n (zero mod n, not zero), and non-units p*2^j for n = p*q, mixed with random units in every warp"""
    from tests.golden import fixtures
    ks = fixtures.load_keyset(0)
    rng = random.Random(0x1417 + bits)
    R, W = 1 << bits, bits // JOB_TPI[bits]
    primes = [ks[0].dk.p, ks[0].dk.q] if bits == 2048 else [ks[0].dk.p, ks[0].dk.q, ks[1].dk.p, ks[1].dk.q]
    pq = 1
    for f in primes:
        pq *= f
    ns = [pq] + co.moduli(bits, JOB_TPI[bits], rng)
    a, m = [], []
    for n in ns:
        special = [1 << j for k in range(JOB_TPI[bits]) for j in (W * k - 1, W * k, W * k + 1) if 0 <= j < bits]
        special += [n - 1, n - 2, R - 1, n + 1, n]
        if 2 * n < R:
            special.append(2 * n)
        if n == pq:
            special += [primes[0] << j for j in (0, 1, 31, 32, W, bits - primes[0].bit_length() - 1)]
        for x in special:
            if 0 <= x < R:
                a.append(x); m.append(n)
                a.append(rng.randrange(1, n)); m.append(n)            # a (likely) unit next to it in the warp
    if len(a) % (32 // JOB_TPI[bits]) == 0:
        a.append(3); m.append(ns[0])

    def inv(x, n):
        try:
            return pow(x, -1, n)
        except ValueError:
            return None

    want = [inv(x, n) for x, n in zip(a, m)]
    assert want.count(None) >= 8
    got = engine.mod_inv(a, m, bits)
    bad = [i for i in range(len(a)) if got[i] != want[i]]
    assert not bad, [(hex(a[i])[:24], hex(m[i])[:24], got[i] is None, want[i] is None) for i in bad[:4]]


# ------------------------------------------------------------------------------------------------ 4/5. N-adic Paillier, every shape
def _nadic_inputs():
    rng = random.Random(0x9ADC)
    ns = []
    for t in (8, 4):
        ns += [n for n in co.moduli(2048, t, rng) if n not in ns]
    cts = co.lane_values(128, 16, rng) + co.lane_values(128, 8, rng)
    cts += [(1 << 4096) - 1, co.rrandomb(4096, rng, True), co.rrandomb(4096, rng, False), co.rrandomb(4096, rng)]
    count = 3 * len(ns) + 7
    idx = [i % len(ns) for i in range(count)]
    c = [cts[(5 * i) % len(cts)] for i in range(count)]
    c2 = [cts[(5 * i + 3) % len(cts)] for i in range(count)]
    msg = co.structured(2048, 8, rng) + co.structured(2048, 4, rng)
    m = [msg[(3 * i) % len(msg)] for i in range(count)]
    r = [msg[(7 * i + 2) % len(msg)] for i in range(count)]
    muls = []
    for kl in (1, 3, 5, 63, 64):
        es = co.exponents(32 * kl, rng)
        k = [es[i % len(es)] for i in range(count)]
        muls.append((kl, k))
    return dict(ns=ns, idx=idx, c=c, c2=c2, m=m, r=r, muls=muls, decrypt=_decrypt_inputs())


def _decrypt_inputs():
    """(key rows, ciphertexts) over the standard key set (rows 0..2) and keys_edge.json (rows 3..): structured 4096-bit
    ciphertexts that are units modulo N (see test_kernel_variants_gpu._decrypt_inputs for why only units)"""
    from tests.golden import fixtures
    rng = random.Random(0xDEC2)
    rows = fixtures.load_keyset(0) + [lk for ks in fixtures.load_edge_keysets() for lk in ks]
    cts = co.lane_values(128, 16, rng) + [(1 << 4096) - 1] + [co.rrandomb(4096, rng, t) for t in (True, False, None, True)]
    idx, cs = [], []
    for i, c in enumerate(cts):
        for row in (i % len(rows), (i * 5 + 1) % len(rows)):
            lk = rows[row]
            if gcd(c, lk.dk.p * lk.dk.q) == 1:
                idx.append(row); cs.append(c)
    return idx, cs


def _nadic_child(inp_path, out_path):
    """Runs in a fresh interpreter with one TECDSA_NADIC_SHAPE: the Paillier batches, outputs to out_path (.npz)."""
    import __graft_entry__ as entry
    pkg = entry.load_package()
    from mpecdsa_b200 import gg20
    from tests.golden import fixtures
    with open(inp_path, "rb") as f:
        I = pickle.load(f)
    L = pkg.ints_to_limbs
    eng = pkg.Engine(0)
    out = {}
    ns, idx = I["ns"], I["idx"]
    for kl, k in I["muls"]:
        out[f"mul{kl}"] = L(eng.paillier_mul(ns, idx, I["c"], k, k_limbs=kl), 128)
    out["add"] = L(eng.paillier_add(ns, idx, I["c"], I["c2"]), 128)
    out["enc"] = L(eng.paillier_encrypt(ns, idx, I["m"], I["r"]), 128)
    ks = gg20.KeySets(eng, [fixtures.load_keyset(0)] + fixtures.load_edge_keysets())
    didx, dcs = I["decrypt"]
    out["dec"] = L(eng.paillier_decrypt(ks.handle, didx, dcs), 64)
    k64 = I["muls"][-1][1]
    out["prof_mul"] = np.array(sorted(eng.profile_step(lambda: eng.paillier_mul(ns, idx, I["c"], k64, k_limbs=64))))
    out["prof_dec"] = np.array(sorted(eng.profile_step(lambda: eng.paillier_decrypt(ks.handle, didx, dcs))))
    ks.free()
    eng.close()
    np.savez(out_path, **out)


@pytest.fixture(scope="module")
def nadic_case(tmp_path_factory):
    from oracle import gg20_oracle as o
    from tests.golden import fixtures
    I = _nadic_inputs()
    path = tmp_path_factory.mktemp("carry-nadic") / "inputs.pkl"
    with open(path, "wb") as f:
        pickle.dump(I, f)
    ns, idx, c = I["ns"], I["idx"], I["c"]
    nn = [n * n for n in ns]
    want = {f"mul{kl}": [pow(cc, kk, nn[i]) for i, cc, kk in zip(idx, c, k)] for kl, k in I["muls"]}
    want["add"] = [x * y % nn[i] for i, x, y in zip(idx, c, I["c2"])]
    want["enc"] = [(1 + mm * ns[i]) * pow(rr, ns[i], nn[i]) % nn[i] for i, mm, rr in zip(idx, I["m"], I["r"])]
    rows = fixtures.load_keyset(0) + [lk for ks in fixtures.load_edge_keysets() for lk in ks]
    want["dec"] = [o.paillier_decrypt(rows[i].dk, x) for i, x in zip(*I["decrypt"])]
    return path, want


def _configs():
    from tests.test_kernel_variants_gpu import CONFIGS
    return CONFIGS


@pytest.mark.parametrize("name", list(_configs()))
def test_paillier_nadic_structured_every_shape(name, nadic_case, tmp_path_factory, pkg):
    """paillier_mul (k_limbs 1, 3, 5, 63, 64), paillier_add, paillier_encrypt over odd-N families with structured
    ciphertexts, exponents and messages, and paillier_decrypt over the standard and edge key sets with structured 4096-bit
    ciphertexts, under each N-adic kernel shape; the per-launch profile shows which instantiation ran."""
    from tests.test_kernel_variants_gpu import VARIANT_ENV
    conf = _configs()[name]
    inp_path, want = nadic_case
    out_path = os.path.join(str(tmp_path_factory.mktemp(f"carry-{name}")), "out.npz")
    env = {k: v for k, v in os.environ.items() if k not in VARIANT_ENV}
    env.update(conf[0])
    code = (f"import sys; sys.path.insert(0, {ROOT!r}); from tests.test_carry_stress_gpu import _nadic_child; "
            f"_nadic_child({str(inp_path)!r}, {out_path!r})")
    flags = ["-s"] if sys.flags.no_user_site else []
    p = subprocess.run([sys.executable, *flags, "-c", code], cwd=ROOT, env=env, timeout=900, capture_output=True, text=True)
    assert p.returncode == 0, f"{name}: child failed (rc={p.returncode})\n{p.stdout[-4000:]}\n{p.stderr[-4000:]}"
    with np.load(out_path) as z:
        got = {k: z[k] for k in z.files}
    _, n64, n32 = conf
    assert {k for k in got["prof_mul"].tolist() if k.startswith("nadic_jobs_kernel")} == {n64}, got["prof_mul"]
    assert {k for k in got["prof_dec"].tolist() if k.startswith("nadic_jobs_kernel")} == {n32}, got["prof_dec"]
    for f, w in want.items():
        g = pkg.limbs_to_ints(got[f])
        bad = [i for i in range(len(w)) if g[i] != w[i]]
        assert not bad, (name, f, bad[:8])


# ------------------------------------------------------------------------------------------------ 6. wide_muladd
def test_wide_muladd_all_ones_and_runs(engine):
    """exact a*b + c with all-ones and run-structured operands at the protocol widths, and above the 132-limb private buffer
    of st::mul_add (its global-memory path)"""
    rng = random.Random(0x3AD)
    for al, bl, cl, ol in ((8, 8, 24, 28), (8, 72, 88, 92), (8, 64, 80, 84), (64, 72, 100, 137), (130, 5, 140, 141),
                           (200, 200, 300, 401)):
        ones = lambda n: (1 << (32 * n)) - 1
        a = [ones(al), ones(al), co.rrandomb(32 * al, rng, True), ones(al), 0, co.rrandomb(32 * al, rng)]
        b = [ones(bl), co.rrandomb(32 * bl, rng, True), ones(bl), 1, ones(bl), co.rrandomb(32 * bl, rng)]
        c = [ones(cl), ones(cl), co.rrandomb(32 * cl, rng, True), ones(cl), ones(cl), co.rrandomb(32 * cl, rng, False)]
        a, b, c = a * 11 + a[:1], b * 11 + b[:1], c * 11 + c[:1]       # 67 operands
        got = engine.wide_muladd(a, b, c, al, bl, cl, ol)
        assert got == [x * y + z for x, y, z in zip(a, b, c)], (al, bl, cl, ol)


def test_wide_muladd_is_exact_or_refused_at_the_width_limit(engine, pkg):
    """a = b = 2^256 - 1 (8 limbs), c = 2^480 - 1 (15 limbs) into 16 limbs: the sum needs 17 limbs, so the widths are
    refused instead of returning the sum minus 2^512.  The tightest widths accepted are exact for all-ones operands."""
    A, C = (1 << 256) - 1, (1 << 480) - 1
    with pytest.raises(pkg.EngineError, match="wide_muladd"):
        engine.wide_muladd([A], [A], [C], 8, 8, 15, 16)
    with pytest.raises(pkg.EngineError, match="wide_muladd"):
        engine.wide_muladd([A], [A], [(1 << 512) - 1], 8, 8, 16, 16)
    for al, bl, cl, ol in ((8, 8, 8, 16), (8, 8, 15, 17), (8, 8, 16, 17), (8, 72, 72, 80), (8, 72, 88, 89), (1, 1, 1, 2)):
        a, b, c = (1 << (32 * al)) - 1, (1 << (32 * bl)) - 1, (1 << (32 * cl)) - 1
        assert engine.wide_muladd([a, a, 0], [b, 1, b], [c, c, c], al, bl, cl, ol) == [a * b + c, a + c, c], (al, bl, cl, ol)


# ------------------------------------------------------------------------------------------------ 7. unit_mod_check
@pytest.mark.parametrize("bits", [2048, 4096])
def test_unit_mod_check_boundaries(engine, keyset, bits):
    """ok iff r < N and gcd(r, N) = 1 for r in {N-1, N, N+1, R-1, 0, 1, lane-aligned values, multiples of a factor}"""
    rng = random.Random(0x0417 + bits)
    R = 1 << bits
    if bits == 2048:
        N, f = keyset[0].dk.p * keyset[0].dk.q, keyset[0].dk.p
    else:
        N, f = keyset[0].dk.p * keyset[0].dk.q * keyset[1].dk.p * keyset[1].dk.q, keyset[1].dk.q
    ns = [N] + co.moduli(bits, JOB_TPI[bits], rng)
    r, m = [], []
    for n in ns:
        for x in [n - 1, n, n + 1, R - 1, 0, 1, n - 2, (n + 1) // 2] + co.lane_values(bits // 32, JOB_TPI[bits], rng):
            if 0 <= x < R:
                r.append(x); m.append(n)
    r += [f, 3 * f, f << 5]; m += [N] * 3
    if len(r) % (32 // JOB_TPI[bits]) == 0:
        r.append(2); m.append(N)
    got = engine.unit_mod_check(r, m, bits)
    assert got == [x < n and gcd(x, n) == 1 for x, n in zip(r, m)]


# ------------------------------------------------------------------------------------------------ 8. modexp chunk boundary
def test_modexp_crosses_the_launch_chunk(engine, pkg, oracle_lib):
    """2^17 + 37 operands (over the 131 072-operand chunk of tecdsa_modexp_batch), 1024-bit structured moduli through
    mod_idx, 1-limb exponents: host buffers and device buffers, every output against GMP"""
    import ctypes
    import torch
    rng = random.Random(0xC4C)
    K, count = 32, (1 << 17) + 37
    ms = _union_moduli(1024, (4, 8, 16), rng)
    npr = np.random.default_rng(0xC4C)
    idx = npr.integers(0, len(ms), size=count).astype(np.uint32)
    base = npr.integers(0, 2**32, size=(count, K), dtype=np.uint32)
    base[::3] = 0xFFFFFFFF                                              # all-ones bases
    base[1::3, : K // 2] = 0                                            # zero low half
    exp = npr.integers(0, 2**32, size=(count, 1), dtype=np.uint32)
    exp[::5] = 0xFFFFFFFF
    M = pkg.ints_to_limbs(ms, K)
    want = np.zeros_like(base)
    threads = max(1, len(os.sched_getaffinity(0)))
    vp = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    oracle_lib.oracle_modexp_batch(vp(base), vp(exp), vp(M), vp(idx), vp(want), ctypes.c_size_t(count), K, 1, threads)
    out = np.zeros_like(base)
    st = np.full(count, 255, np.uint8)
    engine.modexp_raw(1024, 1, base, exp, M, out, st, mod_idx=idx, n_mod=len(ms))
    assert not st.any()
    bad = np.nonzero((out != want).any(axis=1))[0]
    assert bad.size == 0, bad[:8]
    t = lambda a: torch.from_numpy(a.view(np.int32)).cuda()
    dout = torch.zeros_like(t(base))
    dst = torch.full((count,), 255, dtype=torch.uint8, device="cuda")
    engine.modexp_raw(1024, 1, t(base), t(exp), t(M), dout, dst, mod_idx=t(idx), n_mod=len(ms), mem=pkg.DEVICE)
    engine.sync()
    assert dst.sum().item() == 0
    dev = dout.cpu().numpy().view(np.uint32)
    bad = np.nonzero((dev != want).any(axis=1))[0]
    assert bad.size == 0, bad[:8]
