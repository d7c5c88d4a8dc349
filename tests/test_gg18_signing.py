"""CPU tests of GG18 signing as one call (tecdsa_gg18_signing_batch): the party-by-party restatement (tests/gg18_signing_oracle.py)
signs for (1, 3), (2, 5) and (3, 4) keys; the per-element and per-session kernels of csrc/gg18_signing_kernels.cuh and the phase-5c
sender check of csrc/gg18_kernels.cuh run on a host harness against it — the phase-2 sums and statuses, the phase-3 inverse, the
per-sender 5c verdicts and phase 5c with them against its inline checks, and the session stop rule with a failure in every phase —
plus the new export in the header, the package and the Rust FFI."""
import ctypes
import os
import random
import subprocess

import numpy as np
import pytest

import __graft_entry__ as entry
from oracle import gg18_oracle as g18
from oracle import gg20_oracle as o
from oracle.lindell17_oracle import sha256_points_bigint
from tests import gg18_signing_oracle as so
from tests.golden import fixtures

Q, G = o.Q, o.G
HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "host_harness")
OK, INVALID_KEY, NOT_INVERTIBLE, INVALID_SIG, COMMIT = 0, 2, 4, 9, 11


def L(v, k):
    return np.frombuffer(int(v).to_bytes(4 * k, "little"), dtype=np.uint32).copy()


def I(a):
    return int.from_bytes(np.ascontiguousarray(a).tobytes(), "little")


def P_(a):
    return None if a is None else a.ctypes.data_as(ctypes.c_void_p)


def pt16(p):
    return np.zeros(16, np.uint32) if p is None else np.concatenate([L(p[0], 8), L(p[1], 8)])


def from16(a):
    return None if not a.any() else (I(a[:8]), I(a[8:16]))


def rows(vals, k):
    return np.stack([L(v, k) for v in vals])


def make_key(rows_, t, n, rng):
    """a (t, n) key over the Paillier keys of `rows_` (LocalKeys of the fixtures): a fresh degree-t Shamir sharing of a random secret"""
    coef = [rng.randrange(1, Q) for _ in range(t + 1)]
    x = [sum(c * pow(i + 1, k, Q) for k, c in enumerate(coef)) % Q for i in range(n)]
    eks = [o.EncryptionKey(lk.dk.p * lk.dk.q, (lk.dk.p * lk.dk.q) ** 2) for lk in rows_]
    sts = [lk.h1_h2_n_tilde_vec[lk.i - 1] for lk in rows_]
    pks = [o.pt_mul(G, xi) for xi in x]
    return [o.LocalKey(i=i + 1, t=t, n=n, x_i=x[i], dk=rows_[i].dk, pk_vec=pks, paillier_key_vec=eks, h1_h2_n_tilde_vec=sts, y_sum_s=o.pt_mul(G, coef[0]))
            for i in range(n)], coef[0]


def random_signers(keys, s_l, rng):
    """SignerRandomness drawn from `rng` in the ranges of tecdsa_gg18_signing_in"""
    T, out = len(s_l), []
    N = lambda p: keys[p].paillier_key_vec[s_l[p] - 1].n
    for p in range(T):
        r = so.SignerRandomness(**{f: rng.randrange(1, Q) for f in ("k", "gamma", "l", "rho", "heg_s1", "heg_s2", "dlog_nonce")},
                                **{f: rng.getrandbits(256) for f in ("blind", "blind5", "blind5c")}, r_a=rng.randrange(N(p)))
        for j in range(T - 1):
            a = j if j < p else j + 1
            for f in ("beta_tag_gamma", "r_gamma", "beta_tag_w", "r_w"):
                getattr(r, f).append(rng.randrange(N(a)))
            for f in ("nonce_gamma_b", "nonce_gamma_beta", "nonce_w_b", "nonce_w_beta"):
                getattr(r, f).append(rng.randrange(1, Q))
        out.append(r)
    return out


@pytest.fixture(scope="module")
def hg():
    so_path = os.path.join(HERE, "libgg18_signing_host.so")
    src = os.path.join(HERE, "gg18_signing_harness.cpp")
    deps = [src] + [os.path.join(entry.CSRC, f) for f in os.listdir(entry.CSRC) if f.endswith((".cuh", ".h"))] + \
           [os.path.join(entry.ROOT, "include", "tecdsa_b200.h")]
    if not os.path.exists(so_path) or any(os.path.getmtime(s) > os.path.getmtime(so_path) for s in deps):
        subprocess.check_call(["g++", "-O1", "-w", "-I", HERE, "-I", entry.CSRC, "-shared", "-fPIC", "-o", so_path, src])
    lib = ctypes.CDLL(so_path)
    V, I_ = ctypes.c_void_p, ctypes.c_int
    lib.h_session.argtypes = [I_] + [V] * 5 + [I_]
    lib.h_msgb.argtypes = [I_, I_, V, V]
    lib.h_phase2.argtypes = [I_, I_] + [V] * 9
    lib.h_phase3.argtypes = [I_, V, V, V, I_]
    lib.h_round_end.argtypes = [I_, V, V, V, I_]
    lib.h_finish.argtypes = [I_] + [V] * 12 + [I_]
    lib.h_phase5a.argtypes = [V] * 13 + [I_]
    lib.h_phase5c_senders.argtypes = [V] * 7 + [I_]
    lib.h_phase5c.argtypes = [I_] + [V] * 14 + [I_, V]
    lib.h_init()
    return lib


@pytest.mark.parametrize("t,n,s_l", [(1, 3, [3, 1]), (2, 5, [5, 2, 3]), (3, 4, [2, 4, 1, 3])])
def test_oracle_flow_signs(t, n, s_l):
    """sign_session for a (t, n) key and `s_l`: every signer keeps OK, the signature verifies under `cryptography`, and it equals
    k^-1 (m + r x) for the opened secrets (R = k^-1 G with k = sum k_i; s up to low-s normalisation)"""
    from cryptography.hazmat.primitives import hashes
    from cryptography.hazmat.primitives.asymmetric import ec, utils
    rng = random.Random(0x6718 + 16 * t + n)
    fix = [lk for ks in fixtures.load_all_keysets() for lk in ks]
    key, x = make_key(fix[:n], t, n, rng)
    keys = [key[i - 1] for i in s_l]
    rnd = random_signers(keys, s_l, rng)
    m = rng.getrandbits(256) % Q
    res = so.sign_session(keys, s_l, rnd, m)
    assert res.status == [OK] * len(s_l) and res.phase == -1
    r, s, recid = res.signature
    k = sum(v.k for v in rnd) % Q
    assert res.R[0] == o.pt_mul(G, pow(k, -1, Q)) and all(R == res.R[0] for R in res.R)
    assert r == res.R[0][0] % Q and s in (k * (m + r * x) % Q, (-k * (m + r * x)) % Q)
    y = key[0].y_sum_s
    pub = ec.EllipticCurvePublicNumbers(y[0], y[1], ec.SECP256K1()).public_key()
    pub.verify(utils.encode_dss_signature(r, s), m.to_bytes(32, "big"), ec.ECDSA(utils.Prehashed(hashes.SHA256())))


def test_oracle_zero_delta_sum_stops_in_phase_3():
    """sum delta_i = (sum k_i)(sum gamma_i): gamma of the last signer = -(the others') gives NotInvertible for every signer"""
    rng = random.Random(0x0D)
    fix = [lk for ks in fixtures.load_all_keysets() for lk in ks]
    key, _ = make_key(fix[:3], 1, 3, rng)
    rnd = random_signers(key[:2], [1, 2], rng)
    rnd[1].gamma = (-rnd[0].gamma) % Q
    res = so.sign_session(key[:2], [1, 2], rnd, 5)
    assert res.status == [NOT_INVERTIBLE] * 2 and res.phase == 2 and res.signature is None


def _layout(rng, T, n):
    """pairs of the kernel layout: back[(b, v)] = the pair in which element b sends to element v"""
    E = n * T
    back = {}
    for u in range(E):
        for j in range(T - 1):
            back[(u, u - u % T + (j if j < u % T else j + 1))] = j * E + u
    return E, (T - 1) * E, back


def test_phase2_sums_and_statuses(hg):
    """delta_i = k gamma + sum alpha + sum beta and sigma_i = k w + sum mu + sum nu equal phase2_sum of the oracle; a failed get_alpha
    of either half fails its receiver only with InvalidKey; a failed MessageB is charged to its sender with the step's code, the
    gamma half first"""
    rng = random.Random(0x2D18)
    for T in (2, 3, 5):
        n = 3
        E, NP, back = _layout(rng, T, n)
        k, gam, w = ([rng.randrange(1, Q) for _ in range(E)] for _ in range(3))
        alpha = [rng.randrange(Q) for _ in range(2 * NP)]
        beta = [rng.randrange(Q) for _ in range(2 * NP)]
        st_a = np.zeros(2 * NP, np.uint8)
        st_a[back[(1, 0)]] = INVALID_KEY                       # element 0 fails to open element 1's MessageB(gamma)
        st_a[NP + back[(E - 1, E - 2)]] = INVALID_KEY          # element E-2 fails to open element E-1's MessageB(w)
        delta, sigma, cand = np.zeros((E, 8), np.uint32), np.zeros((E, 8), np.uint32), np.zeros(E, np.uint8)
        args = [rows(alpha, 8), rows(beta, 8), rows(k, 8), rows(gam, 8), rows(w, 8)]
        hg.h_phase2(T, E, P_(st_a), *[P_(a) for a in args], P_(delta), P_(sigma), P_(cand))
        for v in range(E):
            peers = [v - v % T + (j if j < v % T else j + 1) for j in range(T - 1)]
            ins = [back[(b, v)] for b in peers]
            outs = [j * E + v for j in range(T - 1)]
            assert I(delta[v]) == g18.phase2_sum(k[v], gam[v], [alpha[t] for t in ins], [beta[t] for t in outs])
            assert I(sigma[v]) == g18.phase2_sum(k[v], w[v], [alpha[NP + t] for t in ins], [beta[NP + t] for t in outs])
            assert cand[v] == (INVALID_KEY if v in (0, E - 2) else OK), (T, v)
        st_b = np.zeros(2 * NP, np.uint8)
        st_b[NP + 2] = 7                                       # element 2: its first peer's MessageB(w) ...
        st_b[(T - 2) * E + 2] = 5                              # ... and its last peer's MessageB(gamma): the gamma half wins
        st_b[NP + (T - 2) * E + E - 1] = 3                     # element E-1: its last peer's MessageB(w)
        cand = np.full(E, 255, np.uint8)
        hg.h_msgb(T, E, P_(st_b), P_(cand))
        assert list(cand) == [5 if u == 2 else 3 if u == E - 1 else OK for u in range(E)], T


def test_phase3_inverse_and_zero_sum(hg):
    rng = random.Random(0x3D)
    T, n = 3, 4
    E = n * T
    delta = [rng.randrange(Q) for _ in range(E)]
    delta[T:2 * T] = [5, Q - 12, 7]                             # session 1 sums to zero
    dinv, cand = np.zeros((E, 8), np.uint32), np.zeros(E, np.uint8)
    hg.h_phase3(T, P_(rows(delta, 8)), P_(dinv), P_(cand), n)
    for s in range(n):
        want = g18.phase3_reconstruct_delta(delta[s * T:(s + 1) * T])
        assert list(cand[s * T:(s + 1) * T]) == [NOT_INVERTIBLE if want is None else OK] * T
        assert all(I(dinv[s * T + p]) == (want or 0) for p in range(T))


def _phase5_session(hg, rng, T):
    """one session of T signers through phase 5a on the harness, with one R for every member (what phase 4 gives a session that
    passed it) and a valid signature's algebra: y = x G, sigma_i shares of k x"""
    E = T
    x, k = rng.randrange(1, Q), [rng.randrange(1, Q) for _ in range(T)]
    ksum = sum(k) % Q
    R = o.pt_mul(G, pow(ksum, -1, Q))
    sig_parts = [rng.randrange(Q) for _ in range(T - 1)]
    sig_parts.append((ksum * x - sum(sig_parts)) % Q)
    m = rng.getrandbits(256) % Q
    s_i = [g18.phase5_local_sig(k[p], m, R, sig_parts[p]) for p in range(T)]
    f = {n: [rng.randrange(1, Q) for _ in range(E)] for n in ("l", "rho", "hs1", "hs2", "dn")}
    f.update({n: [rng.getrandbits(256) for _ in range(E)] for n in ("b5", "b5c")})
    A = {n: rows(v, 8) for n, v in f.items()}
    A["R"] = np.stack([pt16(R)] * E)
    A["y"] = np.stack([pt16(o.pt_mul(G, x))] * E)
    A["m"] = rows([m] * E, 8)
    A["s"] = rows(s_i, 8)
    A["com"], A["vab"], A["heg"], A["dlog"] = (np.zeros((E, w), np.uint32) for w in (8, 48, 48, 40))
    st = np.full(E, 255, np.uint8)
    hg.h_phase5a(P_(A["R"]), P_(A["s"]), P_(A["l"]), P_(A["rho"]), P_(A["b5"]), P_(A["hs1"]), P_(A["hs2"]), P_(A["dn"]), P_(A["com"]), P_(A["vab"]),
                 P_(A["heg"]), P_(A["dlog"]), P_(st), E)
    assert not st.any()
    return A, R, f


def _phase5a_of(A, f, v):
    d, h, g = A["vab"][v], A["heg"][v], A["dlog"][v]
    return g18.Phase5A(I(A["com"][v]), from16(d[:16]), from16(d[16:32]), from16(d[32:48]), f["b5"][v],
                       o.HomoElGamalProof(from16(h[:16]), from16(h[16:32]), I(h[32:40]), I(h[40:48])),
                       o.DLogProof(from16(g[:16]), from16(g[16:32]), I(g[32:40])))


def _run_5c(hg, A, E, verdict):
    com2, ut, st = np.zeros((E, 8), np.uint32), np.zeros((E, 32), np.uint32), np.full(E, 255, np.uint8)
    hg.h_phase5c(E, P_(A["R"]), P_(A["y"]), P_(A["m"]), P_(A["rho"]), P_(A["l"]), P_(A["b5c"]), P_(A["com"]), P_(A["vab"]), P_(A["b5"]), P_(A["heg"]),
                 P_(A["dlog"]), P_(com2), P_(ut), P_(st), E, P_(verdict))
    return com2, ut, st


@pytest.mark.parametrize("tamper", [None, "com", "heg", "dlog"])
def test_phase5c_sender_verdicts(hg, tamper):
    """the per-sender verdicts equal the oracle's three checks (commitment reopens, HomoElGamal proof, DLogProof of rho) on honest
    messages and with one sender's commitment, HomoElGamal proof or DLogProof tampered; k_gg18_phase5c with the verdicts writes
    exactly what its inline checks write (com2, decom2, status), and the status the party-by-party oracle gives every receiver"""
    rng = random.Random(0x5C + [None, "com", "heg", "dlog"].index(tamper))
    T = 4
    A, R, f = _phase5_session(hg, rng, T)
    bad = 2
    if tamper == "com":
        A["com"][bad, 0] ^= 1
    elif tamper == "heg":
        A["heg"][bad, 32:40] = L((I(A["heg"][bad, 32:40]) + 1) % Q, 8)
    elif tamper == "dlog":
        A["dlog"][bad, 32:40] = L((I(A["dlog"][bad, 32:40]) + 1) % Q, 8)
    verdict = np.full(T, 255, np.uint8)
    hg.h_phase5c_senders(P_(A["R"]), P_(A["com"]), P_(A["vab"]), P_(A["b5"]), P_(A["heg"]), P_(A["dlog"]), P_(verdict), T)
    msgs = [_phase5a_of(A, f, v) for v in range(T)]
    for v, a in enumerate(msgs):
        want = o.hash_commitment(sha256_points_bigint([a.V, a.A, a.B]), a.blind) == a.com and o.heg_verify(a.heg, a.A, R, G, a.V, a.B) and \
            o.dlog_verify(a.dlog)
        assert verdict[v] == int(want) and want == (tamper is None or v != bad), (tamper, v)
    inline = _run_5c(hg, A, T, None)
    shared = _run_5c(hg, A, T, verdict)
    for a, b in zip(inline, shared):
        assert a.tobytes() == b.tobytes()
    y, m = from16(A["y"][0]), I(A["m"][0])
    for p in range(T):
        code, out = g18.phase5c(m, R, y, f["rho"][p], f["l"][p], [msgs[x] for x in range(T) if x != p], msgs[p].V, f["b5c"][p])
        assert shared[2][p] == code == (OK if tamper is None or p == bad else COMMIT), (tamper, p)
        if out:
            assert I(shared[0][p]) == out[0] and from16(shared[1][p][:16]) == out[1] and from16(shared[1][p][16:]) == out[2]


def test_stop_rule_with_a_failure_in_every_phase(hg):
    """eight phases (MessageB, get_alpha, 3, 4, 5a, 5c, 5d, output) over the shared stop rule, then the final scatter: a session
    stops at its first failing phase with exactly the failing members' codes, the other members keep OK, later failures are not
    recorded, other sessions are untouched; a stopped session has zero R and signature and complete = 0"""
    rng = random.Random(0x5709)
    T, n = 3, 10
    E = n * T
    codes = [5, INVALID_KEY, NOT_INVERTIBLE, INVALID_KEY, INVALID_KEY, COMMIT, INVALID_KEY, INVALID_SIG]
    plan = {s + 1: (s, [s % T] if s % 2 == 0 else [0, (s + 1) % T]) for s in range(8)}          # session -> (phase, positions)
    plan[9] = (2, list(range(T)))                                                              # phase 3 fails every member
    status, stopped = np.zeros(E, np.uint8), np.zeros(n, np.uint8)
    for ph in range(8):
        cand = np.zeros(E, np.uint8)
        for s, (p0, ps) in plan.items():
            if p0 <= ph:                                   # a failure keeps failing in later phases
                for p in ps:
                    cand[s * T + p] = codes[ph]
        hg.h_round_end(T, P_(cand), P_(status), P_(stopped), n)
    for s in range(n):
        want = [0] * T
        if s in plan:
            for p in plan[s][1]:
                want[p] = codes[plan[s][0]]
        assert status[s * T:(s + 1) * T].tolist() == want, s
    assert stopped.tolist() == [0] + [1] * (n - 1)
    R, r, s_ = (np.array([[rng.randrange(1, 2 ** 32) for _ in range(w)] for _ in range(E)], np.uint32) for w in (16, 8, 8))
    rid = np.array([rng.randrange(2) for _ in range(E)], np.uint8)
    outs = [np.full(E, 255, np.uint8), np.full((E, 16), 7, np.uint32), np.full((n, 8), 7, np.uint32), np.full((n, 8), 7, np.uint32),
            np.full(n, 9, np.uint8), np.full(n, 9, np.uint8)]
    hg.h_finish(T, P_(status), P_(stopped), P_(R), P_(r), P_(s_), P_(rid), *[P_(a) for a in outs], E)
    st_o, R_o, r_o, s_o, rec_o, cm_o = outs
    assert list(st_o) == list(status) and list(cm_o) == [1] + [0] * (n - 1)
    assert (R_o[:T] == R[:T]).all() and not R_o[T:].any()
    assert (r_o[0] == r[0]).all() and (s_o[0] == s_[0]).all() and rec_o[0] == rid[0] and not r_o[1:].any() and not s_o[1:].any() and not rec_o[1:].any()


def test_session_operands(hg):
    """every element gets its session's message and the y of its key set"""
    T, n = 3, 4
    sess = np.array([[s % 2] + [0, 1, 2] for s in range(n)], np.uint32)
    msg = np.arange(n * 8, dtype=np.uint32).reshape(n, 8)
    ytab = np.arange(2 * 16, dtype=np.uint32).reshape(2, 16) + 1000
    m8, y16 = np.zeros((n * T, 8), np.uint32), np.zeros((n * T, 16), np.uint32)
    hg.h_session(T, P_(sess), P_(msg), P_(ytab), P_(m8), P_(y16), n * T)
    for u in range(n * T):
        assert (m8[u] == msg[u // T]).all() and (y16[u] == ytab[(u // T) % 2]).all()


def test_new_export_in_header_package_and_ffi(pkg, tmp_path):
    import re
    hdr = open(os.path.join(entry.ROOT, "include", "tecdsa_b200.h")).read()
    ffi = open(os.path.join(entry.ROOT, "bindings", "rust", "src", "ffi.rs")).read()
    name = "tecdsa_gg18_signing_batch"
    assert re.search(rf"\b{name}\s*\(", hdr) and name in pkg.EXPORTS and f"pub fn {name}(" in ffi
    for struct in ("tecdsa_gg18_signing_in", "tecdsa_gg18_signing_out"):
        assert f"pub struct {struct}" in ffi
    from mpecdsa_b200 import gg18
    body = lambda s: hdr.split(f"}} {s};")[0].split("typedef struct {")[-1]
    assert [f for f, _ in gg18._SigningIn._fields_] == re.findall(r"const uint32_t\* (\w+);", body("tecdsa_gg18_signing_in"))
    assert [f for f, _ in gg18._SigningOut._fields_] == re.findall(r"uint\d+_t\* (\w+);", body("tecdsa_gg18_signing_out"))
    # the stream ids of the header and of the host layer and the restatement
    ids = dict((k, int(v)) for k, v in re.findall(r"TECDSA_RNDS_G18_(\w+) = (\d+)", hdr))
    assert sorted(ids.values()) == list(range(80, 99)) and sorted(gg18.RNDS.values()) == sorted(ids.values()) and gg18.RNDS == so.STREAMS
    # ffi.rs is what the generator writes, and the header compiles as C99 with -Werror
    import importlib.util
    spec = importlib.util.spec_from_file_location("gen_rust_ffi", os.path.join(entry.ROOT, "tools", "gen_rust_ffi.py"))
    gen_ffi = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen_ffi)
    gen_ffi.OUT = str(tmp_path / "ffi.rs")
    gen_ffi.main()
    assert (tmp_path / "ffi.rs").read_text() == ffi
    c = tmp_path / "h.c"
    c.write_text('#include "tecdsa_b200.h"\nint main(void) { tecdsa_gg18_signing_in i; tecdsa_gg18_signing_out o; (void)i; (void)o; '
                 'return TECDSA_RNDS_G18_K == 80 ? 0 : 1; }\n')
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Wextra", "-Werror", "-pedantic", "-I", os.path.join(entry.ROOT, "include"), "-fsyntax-only", str(c)])
