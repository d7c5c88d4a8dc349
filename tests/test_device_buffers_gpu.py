"""Every staged batch entry point (each prototype of include/tecdsa_b200.h that ends in `int mem)`) run on TECDSA_DEVICE buffers
and checked byte for byte against its TECDSA_HOST call.

The HOST path copies each caller buffer to pool scratch (csrc/stage.cuh `Stage`) and copies results back; the DEVICE path hands
the caller's memory to the kernels.  For valid inputs the two must agree exactly, so the library's HOST result (pinned to the
oracle by the rest of the suite, and here again at the first and last element) is the oracle of its DEVICE result.  Each entry of
SPECS below names every argument of one entry point: scalars, and every buffer with its role, element type, row count and row
width, as the header documents them.  Per entry point and batch size (1 and 65: more than one 64-thread block, not a multiple of
the 4 or 8 lane groups of a warp) three runs are compared:

  (a) HOST, numpy buffers;  (b) DEVICE, CUDA buffers on the session context;  (c) DEVICE on a second context on a private stream.

In every run each buffer sits between two 64-byte 0xA5 guards with its data 16-byte aligned; after the call the guards are
untouched, every input (guards included) is unchanged, and every output is identical across the three runs.  The last element
of each batch fills its slots up to the top limb wherever the ABI allows (values >= N^2 for the N-adic jobs, N - 1, q - 1,
2^2048 - 1 ...), so an `S.in` that stages a few bytes too few shows as a HOST/DEVICE difference.  Verifier batches mix accepted
and tampered elements.  Further: chains of DEVICE calls queued on a private stream with one sync at the end, two contexts
interleaved from one thread, and tecdsa_sha256_batch refusing DEVICE buffers.  The coverage test runs without a GPU.
"""
import ctypes
import functools
import os
import random
import re

import numpy as np
import pytest

from oracle import gg20_oracle as o
from oracle import gg18_oracle as g18
from oracle import keygen_oracle as kg
from oracle import lindell17_oracle as l17
from oracle import seeded_sampling as ss
from tests.golden import fixtures

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "tecdsa_b200.h")
HOST, DEVICE, E_UNSUPPORTED = 0, 1, -4
GUARD, FILL_GUARD, FILL_OUT = 64, 0xA5, 0x5A
COUNTS = (1, 65)
Q, Q3 = o.Q, o.Q ** 3
ALPHA_TOP = Q3 - (Q << 256) - 1              # the largest alpha an honest verifier accepts for every challenge (s1 = e a + alpha <= q^3)
SEED = bytes(range(32))
SALT = b"KZen"
ITEMS = (64, 8, 16)                                   # sha256_bigints: item widths of one element
DT = {"u8": np.uint8, "u32": np.uint32, "u64": np.uint64, "i32": np.int32}


# ------------------------------------------------------------------------------------------------ the spec table
def I(n):
    return ("int", n)


def Z(n):
    return ("size", n)


def U64(n):
    return ("u64", n)


def U32(n):
    return ("u32", n)


def HOSTBUF(n):
    """an argument the entry point always reads from host memory, whatever `mem` says"""
    return ("host", n)


KS, NULL = ("ks",), ("null",)


def In(n, width, rows="count", dt="u32"):
    return ("in", n, dt, rows, width)


def Out(n, width, rows="count", dt="u32"):
    return ("out", n, dt, rows, width)


class Spec:
    def __init__(self, fn, args, build, check=None, variant="", host_only=False):
        self.fn, self.args, self.build, self.check, self.host_only = "tecdsa_" + fn, args, build, check, host_only
        self.id = fn + (":" + variant if variant else "")

    def buffers(self, role=None):
        return [a for a in self.args if a[0] in ("in", "out") and (role is None or a[0] == role)]


def _ev(x, sc):
    return x if isinstance(x, int) else int(eval(x, {}, dict(sc)))


def _shape(a, sc):
    return _ev(a[3], sc), _ev(a[4], sc)


SPECS = []


def spec(fn, args, variant="", check=None, host_only=False):
    def deco(build):
        SPECS.append(Spec(fn, args, build, check, variant, host_only))
        return build
    return deco


# ------------------------------------------------------------------------------------------------ values
L = lambda vals, k: np.frombuffer(b"".join(int(v).to_bytes(4 * k, "little") for v in vals), dtype="<u4").reshape(len(vals), k).copy()
ints = lambda a: [int.from_bytes(np.ascontiguousarray(r).tobytes(), "little") for r in a.reshape(a.shape[0], -1)]
pack = lambda p: 0 if p is None else p[0] | (p[1] << 256)
unpack = lambda v: None if v == 0 else (v & ((1 << 256) - 1), v >> 256)
P = lambda pts: L([pack(p) for p in pts], 16)
row_int = lambda a, i: int.from_bytes(np.ascontiguousarray(a[i]).tobytes(), "little")
row_pt = lambda a, i: unpack(row_int(a, i))


class World:
    """The key rows (the standard key set, then an edge key set), the batch's row assignment and a deterministic generator.
    rows_for(n)[-1] is an edge row with a 2047-bit N, so that the last element can carry a ciphertext >= N^2 in 4096 bits."""

    def __init__(self, eng, ksh, keys):
        self.eng, self.ksh, self.keys = eng, ksh, keys
        self.last = next(r for r in (3, 4, 5) if self.N(r).bit_length() == 2047)
        self.host_cache = {}

    def rng(self, tag, n):
        return random.Random(f"{tag}/{n}")

    def rows_for(self, n):
        return [(self.last - (n - 1 - i)) % 6 for i in range(n)]

    def N(self, r):
        return self.keys[r].dk.p * self.keys[r].dk.q

    def ek(self, r):
        n = self.N(r)
        return o.EncryptionKey(n, n * n)

    def dk(self, r):
        return self.keys[r].dk

    def st(self, r):
        lk = self.keys[r]
        return lk.h1_h2_n_tilde_vec[lk.i - 1]

    def unit(self, rng, n):
        while True:
            v = rng.randrange(1, n)
            if v % self.dk_of_n(n)[0] and v % self.dk_of_n(n)[1]:
                return v

    def dk_of_n(self, n):
        for lk in self.keys:
            if lk.dk.p * lk.dk.q == n:
                return lk.dk.p, lk.dk.q
        raise KeyError(n)

    def top_c(self, c, r):
        """c + k N^2 for the largest k that keeps it below 2^4096: a ciphertext that fills its top limb"""
        nn = self.N(r) ** 2
        return c + ((1 << 4096) - 1 - c) // nn * nn

    def host(self, fn, inp, sc, variant=""):
        """outputs of one plain HOST call (inputs of the next entry point are made by the library's own provers)"""
        sp = next(s for s in SPECS if s.fn == "tecdsa_" + fn and s.id.endswith(variant))
        rc, outs = _call(self.eng.lib, self.eng._ctx, self.ksh, sp, inp, sc, HOST, guard=False)
        assert rc == 0, (fn, rc)
        return outs

    def enc(self, rows, m, r):
        n = len(rows)
        return self.host("paillier_encrypt_batch", {"n": L([self.N(x) for x in range(6)], 64), "key_idx": np.array(rows, np.uint32), "m": L(m, 64),
                                              "r": L(r, 64)}, {"n_keys": 6, "count": n}, "idx")["c"]


def scalars(rng, n, top=Q - 1):
    v = [rng.randrange(1, Q) for _ in range(n)]
    v[-1] = top
    return v


def points(rng, n):
    return [o.pt_mul(o.G, rng.randrange(1, Q)) for _ in range(n)]


def tamper(a, n, col=0):
    """flip the low bit of word `col` of every third element (0, 3, ...) short of the last three (the last GG18 session of three
    signers): verifier batches mix accept / reject, and their last element is accepted"""
    a = a.copy()
    for i in range(0, n - 3, 3):
        a[i, col] ^= 1
    return a


# ------------------------------------------------------------------------------------------------ L0
MODIDX = lambda K: [In("modulus", K, "n_mod or count"), In("mod_idx", 1), Z("n_mod")]


@spec("modexp_batch", [I("mod_bits"), I("exp_limbs"), In("base", "mod_bits // 32"), In("exp", "exp_limbs")] + MODIDX("mod_bits // 32") +
      [Out("out", "mod_bits // 32"), Out("status", 1, dt="u8"), Z("count")],
      check=lambda W, i, s, x: row_int(x["out"], s) == pow(row_int(i["base"], s), row_int(i["exp"], s), W.N(W.rows_for(i["_n"])[s])))
def _modexp(W, n):
    rng, rows = W.rng("modexp", n), W.rows_for(n)
    base = [rng.getrandbits(2048) for _ in rows]; base[-1] = (1 << 2048) - 1
    exp = [rng.getrandbits(256) for _ in rows]; exp[-1] = (1 << 256) - 1
    return {"base": L(base, 64), "exp": L(exp, 8), "modulus": L([W.N(r) for r in rows], 64), "mod_idx": None, "_n": n}, \
        {"mod_bits": 2048, "exp_limbs": 8, "n_mod": 0, "count": n}


def _mod_tab(W, n, tag):
    rng, rows = W.rng(tag, n), W.rows_for(n)
    return rng, rows, {"modulus": L([W.N(r) for r in range(6)], 64), "mod_idx": np.array(rows, np.uint32)}


@spec("modmul_batch", [I("mod_bits"), In("a", "mod_bits // 32"), In("b", "mod_bits // 32")] + MODIDX("mod_bits // 32") +
      [Out("out", "mod_bits // 32"), Z("count")],
      check=lambda W, i, s, x: row_int(x["out"], s) == row_int(i["a"], s) * row_int(i["b"], s) % W.N(int(i["mod_idx"][s])))
def _modmul(W, n):
    rng, rows, inp = _mod_tab(W, n, "modmul")
    a = [rng.randrange(W.N(r)) for r in rows]; a[-1] = W.N(rows[-1]) - 1
    b = [rng.randrange(W.N(r)) for r in rows]; b[-1] = W.N(rows[-1]) - 2
    return dict(inp, a=L(a, 64), b=L(b, 64)), {"mod_bits": 2048, "n_mod": 6, "count": n}


def _inv_or_zero(a, m):
    try:
        return pow(a, -1, m), 1
    except ValueError:
        return 0, 0


@spec("modinv_batch", [I("mod_bits"), In("a", "mod_bits // 32")] + MODIDX("mod_bits // 32") + [Out("out", "mod_bits // 32"), Out("ok", 1, dt="u8"), Z("count")],
      check=lambda W, i, s, x: (row_int(x["out"], s), int(x["ok"][s, 0])) == _inv_or_zero(row_int(i["a"], s), W.N(int(i["mod_idx"][s]))))
def _modinv(W, n):
    rng, rows, inp = _mod_tab(W, n, "modinv")
    a = [rng.randrange(1, W.N(r)) if i % 5 != 1 else W.dk(r).p for i, r in enumerate(rows)]    # every fifth from the second: not invertible
    a[-1] = W.N(rows[-1]) - 2
    return dict(inp, a=L(a, 64)), {"mod_bits": 2048, "n_mod": 6, "count": n}


@spec("secp_mul_batch", [In("points", 16), In("scalars", 8), Out("out", 16), Z("count")],
      check=lambda W, i, s, x: row_pt(x["out"], s) == o.pt_mul(row_pt(i["points"], s), row_int(i["scalars"], s) % Q))
def _secp_mul(W, n):
    rng = W.rng("secp_mul", n)
    return {"points": P(points(rng, n)), "scalars": L(scalars(rng, n, (1 << 256) - 1), 8)}, {"count": n}


for _op, _f in (("add", o.pt_add), ("sub", o.pt_sub)):
    @spec(f"secp_{_op}_batch", [In("a", 16), In("b", 16), Out("out", 16), Z("count")],
          check=lambda W, i, s, x, f=_f: row_pt(x["out"], s) == f(row_pt(i["a"], s), row_pt(i["b"], s)))
    def _secp_add(W, n, op=_op):
        rng = W.rng("secp_" + op, n)
        a, b = points(rng, n), points(rng, n)
        if n > 2:
            b[1] = a[1] if op == "sub" else o.pt_neg(a[1])             # the identity as a result
        return {"a": P(a), "b": P(b)}, {"count": n}


@spec("secp_compress_batch", [In("points", 16), Out("out33", 33, dt="u8"), Z("count")],
      check=lambda W, i, s, x: bytes(x["out33"][s]) == o.pt_compress(row_pt(i["points"], s)))
def _compress(W, n):
    return {"points": P(points(W.rng("compress", n), n))}, {"count": n}


def _decompress_check(W, i, s, x):
    enc = bytes(i["in33"][s])
    want = next((p for p in [_lift(enc)] if p is not None), None)
    return (row_pt(x["points"], s), int(x["ok"][s, 0])) == (want, 1 if want else 0)


def _lift(enc):
    if enc[0] not in (2, 3):
        return None
    xx = int.from_bytes(enc[1:], "big")
    if xx >= o.P:
        return None
    y = pow((xx ** 3 + 7) % o.P, (o.P + 1) // 4, o.P)
    if y * y % o.P != (xx ** 3 + 7) % o.P:
        return None
    return (xx, y if y % 2 == enc[0] - 2 else o.P - y)


@spec("secp_decompress_batch", [In("in33", 33, dt="u8"), Out("points", 16), Out("ok", 1, dt="u8"), Z("count")], check=_decompress_check)
def _decompress(W, n):
    rng = W.rng("decompress", n)
    enc = [bytearray(o.pt_compress(p)) for p in points(rng, n)]
    for i in range(0, n - 1, 4):
        enc[i][0] = 5                                                  # malformed prefix
    return {"in33": np.frombuffer(b"".join(enc), np.uint8).reshape(n, 33).copy()}, {"count": n}


_SOPS = {"mul": lambda a, b: a * b % Q, "add": lambda a, b: (a + b) % Q, "sub": lambda a, b: (a - b) % Q}
for _op in _SOPS:
    @spec(f"secp_scalar_{_op}_batch", [In("a", 8), In("b", 8), Out("out", 8), Z("count")],
          check=lambda W, i, s, x, op=_op: row_int(x["out"], s) == _SOPS[op](row_int(i["a"], s) % Q, row_int(i["b"], s) % Q))
    def _sop(W, n, op=_op):
        rng = W.rng("scalar_" + op, n)
        return {"a": L(scalars(rng, n, (1 << 256) - 1), 8), "b": L(scalars(rng, n, (1 << 256) - (1 << 250) - 1), 8)}, {"count": n}


@spec("secp_scalar_inv_batch", [In("a", 8), Out("out", 8), Out("ok", 1, dt="u8"), Z("count")],
      check=lambda W, i, s, x: (row_int(x["out"], s), int(x["ok"][s, 0])) == _inv_or_zero(row_int(i["a"], s) % Q, Q))
def _sinv(W, n):
    a = scalars(W.rng("scalar_inv", n), n, (1 << 256) - 1)
    if n > 2:
        a[1] = Q                                                       # zero mod q
    return {"a": L(a, 8)}, {"count": n}


@spec("secp_scalar_from_bigint_batch", [In("x", "limbs"), I("limbs"), Out("out", 8), Z("count")],
      check=lambda W, i, s, x: row_int(x["out"], s) == row_int(i["x"], s) % Q)
def _from_bigint(W, n):
    rng = W.rng("from_bigint", n)
    x = [rng.getrandbits(2048) for _ in range(n)]; x[-1] = (1 << 2048) - 1
    return {"x": L(x, 64)}, {"limbs": 64, "count": n}


@spec("wide_muladd_batch", [In("a", "a_limbs"), I("a_limbs"), In("b", "b_limbs"), I("b_limbs"), In("c", "c_limbs"), I("c_limbs"),
                            Out("out", "out_limbs"), I("out_limbs"), Z("count")],
      check=lambda W, i, s, x: row_int(x["out"], s) == row_int(i["a"], s) * row_int(i["b"], s) + row_int(i["c"], s))
def _wide(W, n):
    rng = W.rng("wide", n)
    a, b, c = ([rng.getrandbits(32 * k) for _ in range(n)] for k in (8, 64, 64))
    a[-1], b[-1], c[-1] = (1 << 256) - 1, (1 << 2048) - 1, (1 << 2048) - 1
    return {"a": L(a, 8), "b": L(b, 64), "c": L(c, 64)}, {"a_limbs": 8, "b_limbs": 64, "c_limbs": 64, "out_limbs": 76, "count": n}


def _unit_ok(r, n):
    from math import gcd
    return int(r < n and gcd(r, n) == 1)


@spec("unit_mod_check_batch", [I("mod_bits"), In("r", "mod_bits // 32")] + MODIDX("mod_bits // 32") + [Out("ok", 1, dt="u8"), Z("count")],
      check=lambda W, i, s, x: int(x["ok"][s, 0]) == _unit_ok(row_int(i["r"], s), W.N(int(i["mod_idx"][s]))))
def _unit(W, n):
    rng, rows, inp = _mod_tab(W, n, "unit")
    r = [rng.randrange(1, W.N(x)) for x in rows]
    for i in range(1, n - 1, 4):
        r[i] = W.dk(rows[i]).q                                         # shares a factor
    for i in range(2, n - 1, 4):
        r[i] = W.N(rows[i]) + 1                                        # >= N
    r[-1] = W.N(rows[-1]) - 1
    return dict(inp, r=L(r, 64)), {"mod_bits": 2048, "n_mod": 6, "count": n}


@spec("sha256_batch", [In("bytes", "total", rows=1, dt="u8"), In("offsets", 1, rows="count + 1", dt="u64"), Out("digests", 32, dt="u8"), Z("count")],
      host_only=True, check=lambda W, i, s, x: bytes(x["digests"][s]) == __import__("hashlib").sha256(
          bytes(i["bytes"][0, int(i["offsets"][s, 0]):int(i["offsets"][s + 1, 0])])).digest())
def _sha(W, n):
    rng = W.rng("sha", n)
    msgs = [rng.randbytes(rng.randrange(0, 130)) for _ in range(n)]
    msgs[-1] = b"\xff" * 119
    offs = np.zeros((n + 1, 1), np.uint64)
    offs[1:, 0] = np.cumsum([len(m) for m in msgs])
    blob = b"".join(msgs)
    return {"bytes": np.frombuffer(blob, np.uint8).reshape(1, -1).copy(), "offsets": offs}, {"total": len(blob), "count": n}


# ------------------------------------------------------------------------------------------------ L1 Paillier
PKEY = [In("n", 64, "n_keys or count"), In("key_idx", 1), Z("n_keys")]


def _pkey(W, n, with_idx):
    rows = W.rows_for(n)
    if with_idx:
        return rows, {"n": L([W.N(r) for r in range(6)], 64), "key_idx": np.array(rows, np.uint32)}, 6
    return rows, {"n": L([W.N(r) for r in rows], 64), "key_idx": None}, 0


def _ek_elem(W, i, s):
    rows = W.rows_for(i["_n"])
    return W.ek(rows[s])


for _v in ("idx", "rows"):
    @spec("paillier_encrypt_batch", PKEY + [In("m", 64), In("r", 64), Out("c", 128), Z("count")], variant=_v,
          check=lambda W, i, s, x: row_int(x["c"], s) == o.paillier_encrypt(_ek_elem(W, i, s), row_int(i["m"], s), row_int(i["r"], s)))
    def _penc(W, n, v=_v):
        rng = W.rng("penc" + v, n)
        rows, inp, nk = _pkey(W, n, v == "idx")
        m = [rng.randrange(W.N(r)) for r in rows]; m[-1] = W.N(rows[-1]) - 1
        r = [W.unit(rng, W.N(x)) for x in rows]; r[-1] = W.N(rows[-1]) - 1
        return dict(inp, m=L(m, 64), r=L(r, 64), _n=n), {"n_keys": nk, "count": n}


def _ciphers(W, rng, rows, top=True):
    c = [rng.randrange(W.N(r) ** 2) for r in rows]
    if top:
        c[-1] = W.top_c(c[-1], rows[-1])
    return c


for _v in ("idx", "rows"):
    @spec("paillier_mul_batch", PKEY + [In("c", 128), In("k", "k_limbs"), I("k_limbs"), Out("out", 128), Z("count")], variant=_v,
          check=lambda W, i, s, x: row_int(x["out"], s) == pow(row_int(i["c"], s), row_int(i["k"], s), _ek_elem(W, i, s).nn))
    def _pmul(W, n, v=_v):
        rng = W.rng("pmul" + v, n)
        rows, inp, nk = _pkey(W, n, v == "idx")
        k = [rng.getrandbits(256) for _ in rows]; k[-1] = (1 << 256) - 1
        return dict(inp, c=L(_ciphers(W, rng, rows), 128), k=L(k, 8), _n=n), {"n_keys": nk, "k_limbs": 8, "count": n}

    @spec("paillier_add_batch", PKEY + [In("c1", 128), In("c2", 128), Out("out", 128), Z("count")], variant=_v,
          check=lambda W, i, s, x: row_int(x["out"], s) == row_int(i["c1"], s) * row_int(i["c2"], s) % _ek_elem(W, i, s).nn)
    def _padd(W, n, v=_v):
        rng = W.rng("padd" + v, n)
        rows, inp, nk = _pkey(W, n, v == "idx")
        return dict(inp, c1=L(_ciphers(W, rng, rows), 128), c2=L(_ciphers(W, rng, rows), 128), _n=n), {"n_keys": nk, "count": n}


def _pt_cipher(W, rng, rows):
    """valid ciphertexts with their plaintexts; the last element's plaintext is N - 1"""
    m = [rng.randrange(W.N(r)) for r in rows]; m[-1] = W.N(rows[-1]) - 1
    r = [W.unit(rng, W.N(x)) for x in rows]
    return m, r, W.enc(rows, m, r)


@spec("paillier_decrypt_batch", [KS, In("key_row", 1), In("c", 128), Out("m", 64), Z("count")],
      check=lambda W, i, s, x: row_int(x["m"], s) == o.paillier_decrypt(W.dk(int(i["key_row"][s])), row_int(i["c"], s)))
def _pdec(W, n):
    rows = W.rows_for(n)
    _, _, c = _pt_cipher(W, W.rng("pdec", n), rows)
    return {"key_row": np.array(rows, np.uint32), "c": c}, {"count": n}


@spec("paillier_open_batch", [KS, In("key_row", 1), In("c", 128), Out("m", 64), Out("r", 64), Z("count")],
      check=lambda W, i, s, x: (row_int(x["m"], s), row_int(x["r"], s)) == o.paillier_open(W.dk(int(i["key_row"][s])), row_int(i["c"], s)))
def _popen(W, n):
    rows = W.rows_for(n)
    _, _, c = _pt_cipher(W, W.rng("popen", n), rows)
    return {"key_row": np.array(rows, np.uint32), "c": c}, {"count": n}


# ------------------------------------------------------------------------------------------------ L2 range proofs
def _alice_inputs(W, n, tag):
    rng, rows = W.rng(tag, n), W.rows_for(n)
    srows = [(r + 2) % 6 for r in rows]
    a = scalars(rng, n)
    r = [W.unit(rng, W.N(x)) for x in rows]; r[-1] = W.N(rows[-1]) - 1
    c = W.enc(rows, a, r)
    nt = [W.st(x).N for x in srows]
    alpha = [rng.randrange(Q3) for _ in rows]; alpha[-1] = ALPHA_TOP
    beta = [W.unit(rng, W.N(x)) for x in rows]; beta[-1] = W.N(rows[-1]) - 1
    gamma = [rng.randrange(Q3 * t) for t in nt]; gamma[-1] = Q3 * nt[-1] - 1
    rho = [rng.randrange(Q * t) for t in nt]; rho[-1] = Q * nt[-1] - 1
    return {"ek_row": np.array(rows, np.uint32), "st_row": np.array(srows, np.uint32), "a": L(a, 8), "cipher": c, "r": L(r, 64),
            "alpha": L(alpha, 24), "beta": L(beta, 64), "gamma": L(gamma, 88), "rho": L(rho, 72)}, {"count": n}


ALICE_OUT = [("z", 64), ("e", 8), ("s", 64), ("s1", 28), ("s2", 92)]


def _alice_check(W, i, s, x):
    e_r, s_r = int(i["ek_row"][s]), int(i["st_row"][s])
    pf = o.alice_proof_generate(*(row_int(i[k], s) for k in ("a", "cipher")), W.ek(e_r), W.st(s_r), row_int(i["r"], s),
                                *(row_int(i[k], s) for k in ("alpha", "beta", "gamma", "rho")))
    return all(row_int(x[k], s) == getattr(pf, k) for k, _ in ALICE_OUT)


@spec("alice_proof_generate_batch", [KS, In("ek_row", 1), In("st_row", 1), In("a", 8), In("cipher", 128), In("r", 64), In("alpha", 24), In("beta", 64),
                                     In("gamma", 88), In("rho", 72)] + [Out(k, w) for k, w in ALICE_OUT] + [Z("count")], check=_alice_check)
def _alice_gen(W, n):
    return _alice_inputs(W, n, "alice")


def _alice_verify_check(W, i, s, x):
    pf = o.AliceProof(*(row_int(i[k], s) for k, _ in ALICE_OUT))
    return (x["status"][s, 0] == 0) == o.alice_proof_verify(pf, row_int(i["cipher"], s), W.ek(int(i["ek_row"][s])), W.st(int(i["st_row"][s])))


@spec("alice_proof_verify_batch", [KS, In("ek_row", 1), In("st_row", 1), In("cipher", 128)] + [In(k, w) for k, w in ALICE_OUT] +
      [Out("status", 1, dt="u8"), Z("count")], check=_alice_verify_check)
def _alice_ver(W, n):
    inp, sc = _alice_inputs(W, n, "alice-v")
    pf = W.host("alice_proof_generate_batch", inp, sc)
    pf["e"] = tamper(pf["e"], n)
    return dict({k: inp[k] for k in ("ek_row", "st_row", "cipher")}, **pf), sc


PDL_OUT = [("z", 64), ("u1", 16), ("u2", 128), ("u3", 64), ("s1", 28), ("s2", 64), ("s3", 92)]


def _pdl_inputs(W, n, tag):
    rng, rows = W.rng(tag, n), W.rows_for(n)
    srows = [(r + 1) % 6 for r in rows]
    x = scalars(rng, n)
    r = [W.unit(rng, W.N(v)) for v in rows]; r[-1] = W.N(rows[-1]) - 1
    Gp = points(rng, n)
    Qp = [o.pt_mul(g, xx) for g, xx in zip(Gp, x)]
    nt = [W.st(v).N for v in srows]
    alpha = [rng.randrange(Q3) for _ in rows]; alpha[-1] = Q3 - 1
    beta = [rng.randrange(1, W.N(v) - 1) for v in rows]; beta[-1] = W.N(rows[-1]) - 2
    rho = [rng.randrange(Q * t) for t in nt]; rho[-1] = Q * nt[-1] - 1
    gamma = [rng.randrange(Q3 * t) for t in nt]; gamma[-1] = Q3 * nt[-1] - 1
    return {"ek_row": np.array(rows, np.uint32), "st_row": np.array(srows, np.uint32), "x": L(x, 8), "r": L(r, 64), "cipher": W.enc(rows, x, r),
            "Q": P(Qp), "G": P(Gp), "alpha": L(alpha, 24), "beta": L(beta, 64), "rho": L(rho, 72), "gamma": L(gamma, 88)}, {"count": n}


def _pdl_check(W, i, s, x):
    st = W.st(int(i["st_row"][s]))
    pf = o.pdl_prove(row_int(i["x"], s), row_int(i["r"], s), row_int(i["cipher"], s), W.ek(int(i["ek_row"][s])), row_pt(i["Q"], s), row_pt(i["G"], s),
                     st.g, st.ni, st.N, *(row_int(i[k], s) for k in ("alpha", "beta", "rho", "gamma")))
    return all((row_pt(x[k], s) if k == "u1" else row_int(x[k], s)) == getattr(pf, k) for k, _ in PDL_OUT)


@spec("pdl_prove_batch", [KS, In("ek_row", 1), In("st_row", 1), In("x", 8), In("r", 64), In("cipher", 128), In("Q", 16), In("G", 16), In("alpha", 24),
                          In("beta", 64), In("rho", 72), In("gamma", 88)] + [Out(k, w) for k, w in PDL_OUT] + [Z("count")], check=_pdl_check)
def _pdl_prove(W, n):
    return _pdl_inputs(W, n, "pdl")


def _pdl_verify_check(W, i, s, x):
    st = W.st(int(i["st_row"][s]))
    pf = o.PDLwSlackProof(*((row_pt(i[k], s) if k == "u1" else row_int(i[k], s)) for k, _ in PDL_OUT))
    ok = o.pdl_verify(pf, row_int(i["cipher"], s), W.ek(int(i["ek_row"][s])), row_pt(i["Q"], s), row_pt(i["G"], s), st.g, st.ni, st.N)
    return (x["status"][s, 0] == 0) == ok


@spec("pdl_verify_batch", [KS, In("ek_row", 1), In("st_row", 1), In("cipher", 128), In("Q", 16), In("G", 16)] + [In(k, w) for k, w in PDL_OUT] +
      [Out("status", 1, dt="u8"), Z("count")], check=_pdl_verify_check)
def _pdl_ver(W, n):
    inp, sc = _pdl_inputs(W, n, "pdl-v")
    pf = W.host("pdl_prove_batch", inp, sc)
    pf["s1"] = tamper(pf["s1"], n)
    return dict({k: inp[k] for k in ("ek_row", "st_row", "cipher", "Q", "G")}, **pf), sc


BOB_IN = [("b", 8), ("beta_prim", 64), ("r", 64), ("alpha", 24), ("beta", 64), ("gamma", 80), ("ro", 72), ("ro_prim", 88), ("sigma", 72), ("tau", 88)]
BOB_OUT = [("t", 64), ("z", 64), ("e", 8), ("s", 64), ("s1", 28), ("s2", 92), ("t1", 84), ("t2", 92)]


def _bob_inputs(W, n, tag):
    rng, rows = W.rng(tag, n), W.rows_for(n)
    srows = [(r + 4) % 6 for r in rows]
    a_enc = ints(W.enc(rows, scalars(rng, n), [W.unit(rng, W.N(v)) for v in rows]))
    b = scalars(rng, n)
    bp = [rng.randrange(W.N(v) - Q * Q) for v in rows]
    r = [W.unit(rng, W.N(v)) for v in rows]
    enc_bp = ints(W.enc(rows, bp, r))
    mta = [pow(c, bb, W.N(v) ** 2) * e % W.N(v) ** 2 for c, bb, e, v in zip(a_enc, b, enc_bp, rows)]
    nt = [W.st(v).N for v in srows]
    N = [W.N(v) for v in rows]
    vals = {"b": b, "beta_prim": bp, "r": r, "alpha": [rng.randrange(Q3) for _ in rows], "beta": [W.unit(rng, m) for m in N],
            "gamma": [rng.randrange(Q * Q * m) for m in N], "ro": [rng.randrange(Q * t) for t in nt], "ro_prim": [rng.randrange(Q3 * t) for t in nt],
            "sigma": [rng.randrange(Q * t) for t in nt], "tau": [rng.randrange(Q3 * t) for t in nt]}
    vals["alpha"][-1], vals["tau"][-1], vals["ro_prim"][-1], vals["gamma"][-1] = ALPHA_TOP, Q3 * nt[-1] - 1, Q3 * nt[-1] - 1, Q * Q * N[-1] - 1
    inp = {k: L(vals[k], w) for k, w in BOB_IN}
    inp.update(ek_row=np.array(rows, np.uint32), st_row=np.array(srows, np.uint32), a_enc=L(a_enc, 128), mta_enc=L(mta, 128))
    return inp, {"check": 1, "count": n}


def _bob_check(W, i, s, x):
    w, u = o.bob_proof_generate(row_int(i["a_enc"], s), row_int(i["mta_enc"], s), row_int(i["b"], s), row_int(i["beta_prim"], s),
                                W.ek(int(i["ek_row"][s])), W.st(int(i["st_row"][s])), row_int(i["r"], s), True,
                                *(row_int(i[k], s) for k, _ in BOB_IN[3:]))
    return all(row_int(x[k], s) == getattr(w, k) for k, _ in BOB_OUT) and row_pt(x["u"], s) == u


@spec("bob_proof_generate_batch", [KS, In("ek_row", 1), In("st_row", 1), I("check"), In("a_enc", 128), In("mta_enc", 128)] + [In(k, w) for k, w in BOB_IN] +
      [Out(k, w) for k, w in BOB_OUT] + [Out("u", 16), Z("count")], check=_bob_check)
def _bob_gen(W, n):
    return _bob_inputs(W, n, "bob")


def _bob_verify_check(W, i, s, x):
    w = o.BobProof(*(row_int(i[k], s) for k, _ in BOB_OUT))
    ok = o.bob_proof_ext_verify(w, row_pt(i["u"], s), row_int(i["a_enc"], s), row_int(i["mta_out"], s), W.ek(int(i["ek_row"][s])),
                                W.st(int(i["st_row"][s])), row_pt(i["X"], s))
    return (x["status"][s, 0] == 0) == ok


@spec("bob_proof_verify_batch", [KS, In("ek_row", 1), In("st_row", 1), In("a_enc", 128), In("mta_out", 128)] + [In(k, w) for k, w in BOB_OUT] +
      [In("X", 16), In("u", 16), Out("status", 1, dt="u8"), Z("count")], check=_bob_verify_check)
def _bob_ver(W, n):
    inp, sc = _bob_inputs(W, n, "bob-v")
    pf = W.host("bob_proof_generate_batch", inp, sc)
    pf["e"] = tamper(pf["e"], n)
    X = P([o.pt_mul(o.G, v) for v in ints(inp["b"])])
    return dict({k: inp[k] for k in ("ek_row", "st_row", "a_enc")}, mta_out=inp["mta_enc"], X=X, **pf), {"count": n}


# ------------------------------------------------------------------------------------------------ MtA
NST = 2
MTA_A_OUT = [("z", 64), ("e", 8), ("s", 64), ("s1", 28), ("s2", 92)]


def _mta_a_inputs(W, n, tag):
    rng, rows = W.rng(tag, n), W.rows_for(n)
    st_rows = [((r + 1) % 6, (r + 5) % 6) for r in rows]
    a = scalars(rng, n)
    r = [W.unit(rng, W.N(v)) for v in rows]; r[-1] = W.N(rows[-1]) - 1
    pr = []
    for v, sr in zip(rows, st_rows):
        for x in sr:
            nt = W.st(x).N
            pr.append((rng.randrange(Q3), W.unit(rng, W.N(v)), rng.randrange(Q3 * nt), rng.randrange(Q * nt)))
    nt = W.st(st_rows[-1][-1]).N
    pr[-1] = (ALPHA_TOP, W.N(rows[-1]) - 1, Q3 * nt - 1, Q * nt - 1)
    inp = {"ek_row": np.array(rows, np.uint32), "st_rows": np.array(st_rows, np.uint32).reshape(-1, 1), "a": L(a, 8), "r": L(r, 64)}
    for j, (k, w) in enumerate((("alpha", 24), ("beta", 64), ("gamma", 88), ("rho", 72))):
        inp[k] = L([p[j] for p in pr], w)
    return inp, {"n_st": NST, "count": n}


def _mta_a_check(W, i, s, x):
    ek = W.ek(int(i["ek_row"][s]))
    if row_int(x["c"], s) != o.paillier_encrypt(ek, row_int(i["a"], s), row_int(i["r"], s)):
        return False
    j = s * NST + NST - 1
    pf = o.alice_proof_generate(row_int(i["a"], s), row_int(x["c"], s), ek, W.st(int(i["st_rows"][j, 0])), row_int(i["r"], s),
                                *(row_int(i[k], j) for k in ("alpha", "beta", "gamma", "rho")))
    return all(row_int(x[k], j) == getattr(pf, k) for k, _ in MTA_A_OUT)


@spec("mta_message_a_batch", [KS, In("ek_row", 1), In("st_rows", 1, "count * n_st"), I("n_st"), In("a", 8), In("r", 64), In("alpha", 24, "count * n_st"),
                              In("beta", 64, "count * n_st"), In("gamma", 88, "count * n_st"), In("rho", 72, "count * n_st"), Out("c", 128)] +
      [Out(k, w, "count * n_st") for k, w in MTA_A_OUT] + [Z("count")], check=_mta_a_check)
def _mta_a(W, n):
    return _mta_a_inputs(W, n, "mta-a")


MTA_B_IN = [("randomness", 64), ("beta_tag", 64), ("nonce_b", 8), ("nonce_beta", 8)]


def _mta_b_inputs(W, n, tag):
    inp_a, sc = _mta_a_inputs(W, n, tag)
    ma = W.host("mta_message_a_batch", inp_a, sc)
    rng, rows = W.rng(tag + "b", n), W.rows_for(n)
    vals = {"b": scalars(rng, n), "randomness": [W.unit(rng, W.N(v)) for v in rows], "beta_tag": [rng.randrange(W.N(v) - Q * Q) for v in rows],
            "nonce_b": scalars(rng, n), "nonce_beta": scalars(rng, n)}
    vals["randomness"][-1] = W.N(rows[-1]) - 1
    vals["beta_tag"][-1] = W.N(rows[-1]) - Q * Q - 1
    inp = {"ek_row": inp_a["ek_row"], "st_rows": inp_a["st_rows"], "b": L(vals["b"], 8), "c_a": ma["c"]}
    inp.update({k: ma[k] for k, _ in MTA_A_OUT})
    inp.update({k: L(vals[k], w) for k, w in MTA_B_IN})
    return inp, sc, inp_a


def _mta_b_check(W, i, s, x):
    ek = W.ek(int(i["ek_row"][s]))
    pfs = [o.AliceProof(*(row_int(i[k], s * NST + j) for k, _ in MTA_A_OUT)) for j in range(NST)]
    stmts = [W.st(int(i["st_rows"][s * NST + j, 0])) for j in range(NST)]
    res = o.message_b(row_int(i["b"], s), ek, o.MessageA(row_int(i["c_a"], s), pfs), row_int(i["randomness"], s), row_int(i["beta_tag"], s), stmts,
                      row_int(i["nonce_b"], s), row_int(i["nonce_beta"], s))
    if res is None:
        return x["status"][s, 0] == 2
    mb, beta = res
    return x["status"][s, 0] == 0 and row_int(x["c_b"], s) == mb.c and row_int(x["beta"], s) == beta and \
        row_pt(x["b_proof"][:, :16], s) == mb.b_proof.pk and row_int(x["beta_tag_proof"][:, 32:], s) == mb.beta_tag_proof.challenge_response


@spec("mta_message_b_batch", [KS, In("ek_row", 1), In("st_rows", 1, "count * n_st"), I("n_st"), In("b", 8), In("c_a", 128)] +
      [In(k, w, "count * n_st") for k, w in MTA_A_OUT] + [In(k, w) for k, w in MTA_B_IN] +
      [Out("c_b", 128), Out("b_proof", 40), Out("beta_tag_proof", 40), Out("beta", 8), Out("status", 1, dt="u8"), Z("count")], check=_mta_b_check)
def _mta_b(W, n):
    inp, sc, _ = _mta_b_inputs(W, n, "mta-b")
    inp["e"] = tamper(inp["e"], n * NST)                               # an instance with a bad range proof -> ST_INVALID_KEY
    return inp, sc


def _mta_alpha_check(W, i, s, x):
    bp, btp = (i[k][s] for k in ("b_proof", "beta_tag_proof"))
    dl = lambda a: o.DLogProof(unpack(int.from_bytes(a[:16].tobytes(), "little")), unpack(int.from_bytes(a[16:32].tobytes(), "little")),
                               int.from_bytes(a[32:].tobytes(), "little"))
    res = o.verify_proofs_get_alpha(o.MessageB(row_int(i["c_b"], s), dl(bp), dl(btp)), W.dk(int(i["dk_row"][s])), row_int(i["a"], s))
    if res is None:
        return x["status"][s, 0] != 0
    return x["status"][s, 0] == 0 and (row_int(x["alpha"], s), row_int(x["alpha_plain"], s)) == res


@spec("mta_get_alpha_batch", [KS, In("dk_row", 1), In("a", 8), In("c_b", 128), In("b_proof", 40), In("beta_tag_proof", 40), Out("alpha", 8),
                              Out("alpha_plain", 64), Out("status", 1, dt="u8"), Z("count")], check=_mta_alpha_check)
def _mta_alpha(W, n):
    inp_b, sc, inp_a = _mta_b_inputs(W, n, "mta-g")
    mb = W.host("mta_message_b_batch", inp_b, sc)
    return {"dk_row": inp_a["ek_row"], "a": inp_a["a"], "c_b": mb["c_b"], "b_proof": tamper(mb["b_proof"], n, 32),
            "beta_tag_proof": mb["beta_tag_proof"]}, {"count": n}


# ------------------------------------------------------------------------------------------------ key generation
SALTBUF = [In("salt", "salt_len", rows=1, dt="u8"), I("salt_len")]
salt_arr = lambda: np.frombuffer(SALT, np.uint8).reshape(1, -1).copy()


@spec("correct_key_prove_batch", [In("p", 32), In("q", 32)] + SALTBUF + [Out("sigma", 64, "count * 11"), Out("status", 1, dt="u8"), Z("count")],
      check=lambda W, i, s, x: ints(x["sigma"][11 * s:11 * s + 11]) == kg.correct_key_proof(o.DecryptionKey(row_int(i["p"], s), row_int(i["q"], s))))
def _ck_prove(W, n):
    rows = W.rows_for(n)
    return {"p": L([W.dk(r).p for r in rows], 32), "q": L([W.dk(r).q for r in rows], 32), "salt": salt_arr()}, {"salt_len": 4, "count": n}


@spec("correct_key_verify_batch", [In("n", 64), In("sigma", 64, "count * 11")] + SALTBUF + [Out("status", 1, dt="u8"), Z("count")],
      check=lambda W, i, s, x: (x["status"][s, 0] == 0) == kg.correct_key_verify(ints(i["sigma"][11 * s:11 * s + 11]),
                                                                                   o.EncryptionKey(row_int(i["n"], s), row_int(i["n"], s) ** 2)))
def _ck_verify(W, n):
    inp, sc = _ck_prove(W, n)
    sigma = W.host("correct_key_prove_batch", inp, sc)["sigma"]
    for i in range(0, n - 1, 3):
        sigma[11 * i + 5, 0] ^= 1
    return {"n": L([W.N(r) for r in W.rows_for(n)], 64), "sigma": sigma, "salt": inp["salt"]}, sc


def _stmt_rows(W, n):
    return [W.st(r) for r in W.rows_for(n)]


@spec("composite_dlog_prove_batch", [In("n_tilde", 64), In("g", 64), In("ni", 64), In("secret", "secret_limbs"), I("secret_limbs"), In("r", 16),
                                     Out("x", 64), Out("y", "y_limbs"), I("y_limbs"), Z("count")],
      check=lambda W, i, s, x: (lambda pf: (row_int(x["x"], s), row_int(x["y"], s)) == (pf.x, pf.y))(
          kg.composite_dlog_prove(o.DLogStatement(*(row_int(i[k], s) for k in ("n_tilde", "g", "ni"))), row_int(i["secret"], s), row_int(i["r"], s))))
def _cd_prove(W, n):
    rng, sts = W.rng("cd", n), _stmt_rows(W, n)
    sec = [rng.getrandbits(2048) for _ in sts]; sec[-1] = (1 << 2048) - 1
    r = [rng.getrandbits(512) for _ in sts]; r[-1] = (1 << 512) - 1
    return {"n_tilde": L([s.N for s in sts], 64), "g": L([s.g for s in sts], 64), "ni": L([s.ni for s in sts], 64), "secret": L(sec, 64),
            "r": L(r, 16)}, {"secret_limbs": 64, "y_limbs": 76, "count": n}


@spec("composite_dlog_verify_batch", [In("n_tilde", 64), In("g", 64), In("ni", 64), In("x", 64), In("y", "y_limbs"), I("y_limbs"), Out("status", 1, dt="u8"), Z("count")],
      check=lambda W, i, s, x: (x["status"][s, 0] == 0) == kg.composite_dlog_verify(
          kg.CompositeDLogProof(row_int(i["x"], s), row_int(i["y"], s)), o.DLogStatement(*(row_int(i[k], s) for k in ("n_tilde", "g", "ni")))))
def _cd_verify(W, n):
    """proofs for the key-generation statements (N~, h1, h2) with the secret phi - xhi, so that h1^-secret = h2 and honest proofs verify"""
    raw = [p for ks in fixtures.edge_keysets_raw() for p in ks["parties"]]
    sel = [raw[i % len(raw)] for i in range(n)]
    H = lambda r, k: int(r[k], 16)
    rng = W.rng("cd-v", n)
    inp = {"n_tilde": L([H(r, "n_tilde") for r in sel], 64), "g": L([H(r, "h1") for r in sel], 64), "ni": L([H(r, "h2") for r in sel], 64),
           "secret": L([(H(r, "p_tilde") - 1) * (H(r, "q_tilde") - 1) - H(r, "xhi") for r in sel], 64), "r": L([rng.getrandbits(512) for _ in sel], 16)}
    sc = {"secret_limbs": 64, "y_limbs": 76, "count": n}
    pf = W.host("composite_dlog_prove_batch", inp, sc)
    return {k: inp[k] for k in ("n_tilde", "g", "ni")} | {"x": pf["x"], "y": tamper(pf["y"], n)}, {"y_limbs": 76, "count": n}


@spec("vss_share_batch", [I("t"), I("n_shares"), In("coefficients", 8, "count * (t + 1)"), Out("shares", 8, "count * n_shares"),
                          Out("commitments", 16, "count * (t + 1)"), Z("count")],
      check=lambda W, i, s, x: (lambda v: ints(x["shares"][3 * s:3 * s + 3]) == v[1] and [unpack(c) for c in ints(x["commitments"][2 * s:2 * s + 2])] ==
                                v[0].commitments)(kg.vss_share(1, 3, row_int(i["coefficients"], 2 * s), [row_int(i["coefficients"], 2 * s + 1)])))
def _vss_share(W, n):
    c = scalars(W.rng("vss", n), 2 * n, (1 << 256) - 1)
    return {"coefficients": L(c, 8)}, {"t": 1, "n_shares": 3, "count": n}


def _vss_validate_check(W, i, s, x):
    vss = kg.VerifiableSS(1, 3, [unpack(c) for c in ints(i["commitments"][2 * s:2 * s + 2])])
    return (x["status"][s, 0] == 0) == kg.vss_validate_share(vss, row_int(i["share"], s), int(i["index"][s, 0]))


@spec("vss_validate_share_batch", [In("commitments", 16, "count * n_commitments"), I("n_commitments"), In("share", 8), In("index", 1),
                                   Out("status", 1, dt="u8"), Z("count")], check=_vss_validate_check)
def _vss_validate(W, n):
    inp, sc = _vss_share(W, n)
    out = W.host("vss_share_batch", inp, sc)
    idx = [1 + i % 3 for i in range(n)]
    share = np.stack([out["shares"][3 * i + idx[i] - 1] for i in range(n)])
    return {"commitments": out["commitments"], "share": tamper(share, n), "index": np.array(idx, np.uint32).reshape(-1, 1)}, {"n_commitments": 2, "count": n}


def _h1h2_check(W, i, s, x):
    want = kg.h1_h2_n_tilde(*(row_int(i[k], s) for k in ("p_t", "q_t", "h1", "xhi")))
    return x["status"][s, 0] == 0 and [row_int(x[k], s) for k in ("n_tilde", "h2", "xhi_neg", "xhi_inv_neg")] == [want[0], want[2], want[3], want[4]]


@spec("h1_h2_n_tilde_batch", [In("p_t", 32), In("q_t", 32), In("h1", 64), In("xhi", 64), Out("n_tilde", 64), Out("h2", 64), Out("xhi_neg", 64),
                              Out("xhi_inv_neg", 64), Out("status", 1, dt="u8"), Z("count")], check=_h1h2_check)
def _h1h2(W, n):
    raw = [p for ks in fixtures.edge_keysets_raw() for p in ks["parties"]]
    sel = [raw[i % len(raw)] for i in range(n)]
    H = lambda k: [int(r[k], 16) for r in sel]
    return {"p_t": L(H("p_tilde"), 32), "q_t": L(H("q_tilde"), 32), "h1": L(H("h1"), 64), "xhi": L(H("xhi"), 64)}, {"count": n}


# ------------------------------------------------------------------------------------------------ sigma proofs, hashes
def _ddh_inputs(W, n, tag):
    rng = W.rng(tag, n)
    x = scalars(rng, n)
    g1, g2 = points(rng, n), points(rng, n)
    return {"x": L(x, 8), "g1": P(g1), "h1": P([o.pt_mul(g, v) for g, v in zip(g1, x)]), "g2": P(g2),
            "h2": P([o.pt_mul(g, v) for g, v in zip(g2, x)]), "nonce": L(scalars(rng, n), 8)}, {"count": n}


DDH = ("g1", "h1", "g2", "h2")


@spec("ecddh_prove_batch", [In("x", 8)] + [In(k, 16) for k in DDH] + [In("nonce", 8), Out("proof", 40), Z("count")],
      check=lambda W, i, s, x: (lambda pf: row_int(x["proof"], s) == pack(pf.a1) | pack(pf.a2) << 512 | pf.z << 1024)(
          o.ecddh_prove(row_int(i["x"], s), *(row_pt(i[k], s) for k in DDH), row_int(i["nonce"], s))))
def _ddh_prove(W, n):
    return _ddh_inputs(W, n, "ddh")


def _ddh_pf(a, s):
    v = row_int(a, s)
    return o.ECDDHProof(unpack(v & ((1 << 512) - 1)), unpack((v >> 512) & ((1 << 512) - 1)), v >> 1024)


@spec("ecddh_verify_batch", [In("proof", 40)] + [In(k, 16) for k in DDH] + [Out("status", 1, dt="u8"), Z("count")],
      check=lambda W, i, s, x: (x["status"][s, 0] == 0) == o.ecddh_verify(_ddh_pf(i["proof"], s), *(row_pt(i[k], s) for k in DDH)))
def _ddh_verify(W, n):
    inp, sc = _ddh_inputs(W, n, "ddh-v")
    pf = W.host("ecddh_prove_batch", inp, sc)["proof"]
    return {"proof": tamper(pf, n, 32)} | {k: inp[k] for k in DDH}, sc


def _dlog_pf(a, s):
    v = row_int(a, s)
    return o.DLogProof(unpack(v & ((1 << 512) - 1)), unpack((v >> 512) & ((1 << 512) - 1)), v >> 1024)


@spec("dlog_prove_batch", [In("sk", 8), In("nonce", 8), Out("proof", 40), Z("count")],
      check=lambda W, i, s, x: _dlog_pf(x["proof"], s) == o.dlog_prove(row_int(i["sk"], s), row_int(i["nonce"], s)))
def _dlog_prove(W, n):
    rng = W.rng("dlog", n)
    return {"sk": L(scalars(rng, n), 8), "nonce": L(scalars(rng, n), 8)}, {"count": n}


@spec("dlog_verify_batch", [In("proof", 40), Out("status", 1, dt="u8"), Z("count")],
      check=lambda W, i, s, x: (x["status"][s, 0] == 0) == o.dlog_verify(_dlog_pf(i["proof"], s)))
def _dlog_verify(W, n):
    inp, sc = _dlog_prove(W, n)
    return {"proof": tamper(W.host("dlog_prove_batch", inp, sc)["proof"], n, 32)}, sc


def _ped_pf(com, pf, s):
    v = row_int(pf, s)
    f = lambda off, w: (v >> (32 * off)) & ((1 << (32 * w)) - 1)
    return o.PedersenProof(f(0, 8), unpack(f(8, 16)), unpack(f(24, 16)), row_pt(com, s), f(40, 8), f(48, 8))


PED = ("m", "r", "s1", "s2")


@spec("pedersen_prove_batch", [In(k, 8) for k in PED] + [Out("com", 16), Out("proof", 64), Z("count")],
      check=lambda W, i, s, x: _ped_pf(x["com"], x["proof"], s) == o.pedersen_prove(*(row_int(i[k], s) for k in PED)))
def _ped_prove(W, n):
    rng = W.rng("ped", n)
    return {k: L(scalars(rng, n), 8) for k in PED}, {"count": n}


@spec("pedersen_verify_batch", [In("com", 16), In("proof", 64), Out("status", 1, dt="u8"), Z("count")],
      check=lambda W, i, s, x: (x["status"][s, 0] == 0) == o.pedersen_verify(_ped_pf(i["com"], i["proof"], s)))
def _ped_verify(W, n):
    inp, sc = _ped_prove(W, n)
    out = W.host("pedersen_prove_batch", inp, sc)
    return {"com": out["com"], "proof": tamper(out["proof"], n, 40)}, sc


HEG = ("G", "D", "E")


def _heg_inputs(W, n, tag):
    rng = W.rng(tag, n)
    x, r = scalars(rng, n), scalars(rng, n)
    Gp = points(rng, n)
    D = [o.pt_add(o.pt_mul(o.H2, a), o.pt_mul(o.G, b)) for a, b in zip(x, r)]
    E = [o.pt_mul(g, b) for g, b in zip(Gp, r)]
    return {"G": P(Gp), "D": P(D), "E": P(E), "x": L(x, 8), "r": L(r, 8), "s1": L(scalars(rng, n), 8), "s2": L(scalars(rng, n), 8)}, {"count": n}


def _heg_pf(a, s):
    v = row_int(a, s)
    return o.HomoElGamalProof(unpack(v & ((1 << 512) - 1)), unpack((v >> 512) & ((1 << 512) - 1)), (v >> 1024) & ((1 << 256) - 1), v >> 1280)


@spec("heg_prove_batch", [In(k, 16) for k in HEG] + [In(k, 8) for k in ("x", "r", "s1", "s2")] + [Out("proof", 48), Z("count")],
      check=lambda W, i, s, x: _heg_pf(x["proof"], s) == o.heg_prove(row_int(i["x"], s), row_int(i["r"], s), row_pt(i["G"], s), o.H2, o.G,
                                                                     row_pt(i["D"], s), row_pt(i["E"], s), row_int(i["s1"], s), row_int(i["s2"], s)))
def _heg_prove(W, n):
    return _heg_inputs(W, n, "heg")


@spec("heg_verify_batch", [In(k, 16) for k in HEG] + [In("proof", 48), Out("status", 1, dt="u8"), Z("count")],
      check=lambda W, i, s, x: (x["status"][s, 0] == 0) == o.heg_verify(_heg_pf(i["proof"], s), row_pt(i["G"], s), o.H2, o.G, row_pt(i["D"], s), row_pt(i["E"], s)))
def _heg_verify(W, n):
    inp, sc = _heg_inputs(W, n, "heg-v")
    return {k: inp[k] for k in HEG} | {"proof": tamper(W.host("heg_prove_batch", inp, sc)["proof"], n, 32)}, sc


@spec("sha256_bigints_batch", [In("data", sum(ITEMS)), HOSTBUF("item_limbs"), I("n_items"), Out("digest", 8), Z("count")],
      check=lambda W, i, s, x: row_int(x["digest"], s) == o.sha256_bigints(
          [int.from_bytes(i["data"][s, a:a + w].tobytes(), "little") for a, w in zip((0, 64, 72), ITEMS)]))
def _sha_bigints(W, n):
    rng = W.rng("shab", n)
    rows = [[rng.getrandbits(32 * w - rng.randrange(64)) for w in ITEMS] for _ in range(n)]
    rows[-1] = [(1 << (32 * w)) - 1 for w in ITEMS]
    return {"data": np.concatenate([L([r[j] for r in rows], w) for j, w in enumerate(ITEMS)], axis=1), "item_limbs": np.array(ITEMS, np.int32)}, \
        {"n_items": len(ITEMS), "count": n}


@spec("hash_commitment_batch", [In("points", 16), In("blind", 8), Out("com", 8), Z("count")],
      check=lambda W, i, s, x: row_int(x["com"], s) == o.hash_commitment(o.bn_from_bytes(o.pt_compress(row_pt(i["points"], s))), row_int(i["blind"], s)))
def _hcom(W, n):
    rng = W.rng("hcom", n)
    b = [rng.getrandbits(256) for _ in range(n)]; b[-1] = (1 << 256) - 1
    return {"points": P(points(rng, n)), "blind": L(b, 8)}, {"count": n}


# ------------------------------------------------------------------------------------------------ Lindell-2017
EPH_IN = ("secret_share", "nonce", "pk_blind", "zk_pok_blind")
EPH_OUT = [("public_share", 16), ("c_point", 16), ("proof", 40), ("pk_commitment", 8), ("zk_pok_commitment", 8)]


def _eph_check(W, i, s, x):
    e = l17.eph_create(*(row_int(i[k], s) for k in EPH_IN))
    return (row_pt(x["public_share"], s), row_pt(x["c_point"], s), _ddh_pf(x["proof"], s), row_int(x["pk_commitment"], s),
            row_int(x["zk_pok_commitment"], s)) == (e.public_share, e.c, e.proof, e.pk_commitment, e.zk_pok_commitment)


@spec("l17_eph_create_batch", [In(k, 8) for k in EPH_IN] + [Out(k, w) for k, w in EPH_OUT] + [Z("count")], check=_eph_check)
def _eph_create(W, n):
    rng = W.rng("eph", n)
    return {"secret_share": L(scalars(rng, n), 8), "nonce": L(scalars(rng, n), 8), "pk_blind": L(scalars(rng, n, (1 << 256) - 1), 8),
            "zk_pok_blind": L(scalars(rng, n, (1 << 256) - 1), 8)}, {"count": n}


def _eph_verify_check(W, i, s, x):
    msg = l17.EphFirst(row_pt(i["public_share"], s), row_pt(i["c_point"], s), _ddh_pf(i["proof"], s), row_int(i["pk_commitment"], s),
                       row_int(i["zk_pok_commitment"], s))
    return (x["status"][s, 0] == 0) == l17.p1_eph_verify(msg, row_int(i["pk_blind"], s), row_int(i["zk_pok_blind"], s))


@spec("l17_eph_verify_batch", [In("public_share", 16), In("c_point", 16), In("proof", 40), In("pk_blind", 8), In("zk_pok_blind", 8),
                               In("pk_commitment", 8), In("zk_pok_commitment", 8), Out("status", 1, dt="u8"), Z("count")], check=_eph_verify_check)
def _eph_verify(W, n):
    inp, sc = _eph_create(W, n)
    out = W.host("l17_eph_create_batch", inp, sc)
    return {k: out[k] for k in ("public_share", "c_point", "proof", "pk_commitment")} | {
        "zk_pok_commitment": tamper(out["zk_pok_commitment"], n), "pk_blind": inp["pk_blind"], "zk_pok_blind": inp["zk_pok_blind"]}, sc


L17_PS_IN = [("c_key", 128), ("x2", 8), ("k2", 8), ("eph_other_public", 16), ("message", 8), ("rho", 16), ("randomness", 64)]


def _l17_ps_inputs(W, n, tag):
    rng = W.rng(tag, n)
    rows, key, nk = _pkey(W, n, True)
    x1 = scalars(rng, n)
    c_key = W.enc(rows, x1, [W.unit(rng, W.N(v)) for v in rows])
    m = [rng.getrandbits(256) for _ in rows]; m[-1] = (1 << 256) - 1
    rho = [rng.randrange(Q * Q) for _ in rows]; rho[-1] = Q * Q - 1
    rnd = [W.unit(rng, W.N(v)) for v in rows]; rnd[-1] = W.N(rows[-1]) - 1
    k1 = scalars(rng, n)
    inp = dict(key, c_key=c_key, x2=L(scalars(rng, n), 8), k2=L(scalars(rng, n), 8), eph_other_public=P([o.pt_mul(o.G, k) for k in k1]),
               message=L(m, 8), rho=L(rho, 16), randomness=L(rnd, 64), _n=n)
    return inp, {"n_keys": nk, "count": n}, k1


def _l17_ps_check(W, i, s, x):
    want = l17.p2_partial_sig(_ek_elem(W, i, s), *(row_pt(i[k], s) if k == "eph_other_public" else row_int(i[k], s) for k, _ in L17_PS_IN))
    return x["status"][s, 0] == 0 and row_int(x["c3"], s) == want


@spec("l17_partial_sig_batch", PKEY + [In(k, w) for k, w in L17_PS_IN] + [Out("c3", 128), Out("status", 1, dt="u8"), Z("count")], check=_l17_ps_check)
def _l17_ps(W, n):
    return _l17_ps_inputs(W, n, "l17ps")[:2]


def _l17_sign_check(W, i, s, x):
    want = l17.p1_sign(W.dk(int(i["key_row"][s])), row_int(i["c3"], s), row_int(i["k1"], s), row_pt(i["eph_other_public"], s))
    return x["status"][s, 0] == 0 and (row_int(x["sig_r"], s), row_int(x["sig_s"], s), int(x["recid"][s, 0])) == want


@spec("l17_sign_batch", [KS, In("key_row", 1), In("c3", 128), In("k1", 8), In("eph_other_public", 16), Out("sig_r", 8), Out("sig_s", 8),
                         Out("recid", 1, dt="u8"), Out("status", 1, dt="u8"), Z("count")], check=_l17_sign_check)
def _l17_sign(W, n):
    inp, sc, k1 = _l17_ps_inputs(W, n, "l17s")
    c3 = W.host("l17_partial_sig_batch", inp, sc)["c3"]
    k2 = ints(inp["k2"])
    return {"key_row": inp["key_idx"], "c3": c3, "k1": L(k1, 8), "eph_other_public": P([o.pt_mul(o.G, k) for k in k2])}, {"count": n}


def _ecdsa(rng, n):
    x, k, m = scalars(rng, n), scalars(rng, n), [rng.getrandbits(256) for _ in range(n)]
    rs = []
    for xx, kk, mm in zip(x, k, m):
        r = o.pt_mul(o.G, kk)[0] % Q
        s = pow(kk, -1, Q) * (mm % Q + r * xx) % Q
        rs.append((r, min(s, Q - s)))
    return x, m, rs


@spec("l17_verify_batch", [In("sig_r", 8), In("sig_s", 8), In("pubkey", 16), In("message", 8), Out("status", 1, dt="u8"), Z("count")],
      check=lambda W, i, s, x: (x["status"][s, 0] == 0) == l17.verify(row_int(i["sig_r"], s), row_int(i["sig_s"], s), row_pt(i["pubkey"], s), row_int(i["message"], s)))
def _l17_verify(W, n):
    x, m, rs = _ecdsa(W.rng("l17v", n), n)
    return {"sig_r": L([r for r, _ in rs], 8), "sig_s": L([s for _, s in rs], 8), "pubkey": P([o.pt_mul(o.G, v) for v in x]),
            "message": tamper(L(m, 8), n)}, {"count": n}


ZK_V1_IN = [("ciphertext", 128), ("Q", 16), ("a", 8), ("b", 16), ("randomness", 64), ("blindness", 8)]


def _zk_inputs(W, n, tag):
    rng = W.rng(tag, n)
    rows, key, nk = _pkey(W, n, True)
    x1 = scalars(rng, n, Q - 2)                                        # not q - 1: with a = q - 1, b = q^2 - 1 that puts a Q + b G at infinity
    a = [rng.randrange(Q) for _ in rows]; a[-1] = Q - 1
    b = [rng.randrange(Q * Q) for _ in rows]; b[-1] = Q * Q - 1
    rnd = [W.unit(rng, W.N(v)) for v in rows]; rnd[-1] = W.N(rows[-1]) - 1
    inp = dict(key, ciphertext=W.enc(rows, x1, [W.unit(rng, W.N(v)) for v in rows]), Q=P([o.pt_mul(o.G, v) for v in x1]), a=L(a, 8), b=L(b, 16),
               randomness=L(rnd, 64), blindness=L(scalars(rng, n, (1 << 256) - 1), 8), _n=n)
    return inp, {"n_keys": nk, "count": n}, x1


def _zk_v1_check(W, i, s, x):
    st = l17.pdl_verifier_message1(_ek_elem(W, i, s), row_int(i["ciphertext"], s), row_pt(i["Q"], s), *(row_int(i[k], s) for k in ("a", "b", "randomness", "blindness")))
    return x["status"][s, 0] == 0 and (row_int(x["c_tag"], s), row_int(x["c_tag_tag"], s), row_pt(x["q_tag"], s)) == (st.c_tag, st.c_tag_tag, st.q_tag)


@spec("zkpdl_verifier_message1_batch", PKEY + [In(k, w) for k, w in ZK_V1_IN] + [Out("c_tag", 128), Out("c_tag_tag", 8), Out("q_tag", 16),
                                                                                Out("status", 1, dt="u8"), Z("count")], check=_zk_v1_check)
def _zk_v1(W, n):
    return _zk_inputs(W, n, "zkv1")[:2]


def _zk_chain(W, n, tag):
    inp, sc, x1 = _zk_inputs(W, n, tag)
    v1 = W.host("zkpdl_verifier_message1_batch", inp, sc)
    p1_in = {"key_row": inp["key_idx"], "c_tag": v1["c_tag"], "blindness": inp["blindness"]}
    return inp, x1, v1, p1_in


def _zk_p1_check(W, i, s, x):
    want = l17.pdl_prover_message1(W.dk(int(i["key_row"][s])), row_int(i["c_tag"], s), row_int(i["blindness"], s))
    return x["status"][s, 0] == 0 and (row_int(x["c_hat"], s), row_pt(x["q_hat"], s), row_int(x["alpha"], s)) == want


@spec("zkpdl_prover_message1_batch", [KS, In("key_row", 1), In("c_tag", 128), In("blindness", 8), Out("c_hat", 8), Out("q_hat", 16), Out("alpha", 64),
                                      Out("status", 1, dt="u8"), Z("count")], check=_zk_p1_check)
def _zk_p1(W, n):
    return _zk_chain(W, n, "zkp1")[3], {"count": n}


@spec("zkpdl_prover_message2_batch", [In("x1", 8), In("alpha", 64), In("c_tag_tag", 8), In("a", 8), In("b", 16), In("blindness", 8), Out("status", 1, dt="u8"), Z("count")],
      check=lambda W, i, s, x: (x["status"][s, 0] == 0) == l17.pdl_prover_message2(*(row_int(i[k], s) for k in ("x1", "alpha", "c_tag_tag", "a", "b", "blindness"))))
def _zk_p2(W, n):
    inp, x1, v1, p1_in = _zk_chain(W, n, "zkp2")
    p1 = W.host("zkpdl_prover_message1_batch", p1_in, {"count": n})
    return {"x1": L(x1, 8), "alpha": p1["alpha"], "c_tag_tag": tamper(v1["c_tag_tag"], n), "a": inp["a"], "b": inp["b"], "blindness": inp["blindness"]}, {"count": n}


@spec("zkpdl_verifier_finalize_batch", [In("c_hat", 8), In("q_hat", 16), In("blindness", 8), In("q_tag", 16), Out("status", 1, dt="u8"), Z("count")],
      check=lambda W, i, s, x: (x["status"][s, 0] == 0) == l17.pdl_verifier_finalize(row_int(i["c_hat"], s), row_pt(i["q_hat"], s), row_int(i["blindness"], s),
                                                                                      row_pt(i["q_tag"], s)))
def _zk_fin(W, n):
    inp, x1, v1, p1_in = _zk_chain(W, n, "zkfin")
    p1 = W.host("zkpdl_prover_message1_batch", p1_in, {"count": n})
    return {"c_hat": tamper(p1["c_hat"], n), "q_hat": p1["q_hat"], "blindness": inp["blindness"], "q_tag": v1["q_tag"]}, {"count": n}


# ------------------------------------------------------------------------------------------------ GG18 signing phases
PARTIES = 3


@functools.lru_cache(maxsize=None)
def _gg18_world(n):
    """n sessions of PARTIES signers, element u = session * PARTIES + party: R = k^-1 G with k = sum k_i, sum sigma_i = k x,
    s_i = m k_i + r sigma_i; phase-4 inputs with delta_inv = k^-1 / sum gamma_j, so that delta_inv * sum g^gamma_j = R."""
    rng = random.Random(f"gg18/{n}")
    E = n * PARTIES
    w = {k: [] for k in ("k", "gamma", "sigma", "R", "y", "m", "delta_inv", "blind")}
    for _ in range(n):
        k = [rng.randrange(1, Q) for _ in range(PARTIES)]
        gam = [rng.randrange(1, Q) for _ in range(PARTIES)]
        x = rng.randrange(1, Q)
        kk = sum(k) % Q
        sig = [rng.randrange(Q) for _ in range(PARTIES - 1)]
        sig.append((kk * x - sum(sig)) % Q)
        R = o.pt_mul(o.G, pow(kk, -1, Q))
        dinv = pow(kk, -1, Q) * pow(sum(gam) % Q, -1, Q) % Q
        m = rng.getrandbits(256)
        w["k"] += k; w["gamma"] += gam; w["sigma"] += sig; w["R"] += [R] * PARTIES; w["y"] += [o.pt_mul(o.G, x)] * PARTIES
        w["m"] += [m] * PARTIES; w["delta_inv"] += [dinv] * PARTIES
    w["blind"] = [rng.getrandbits(256) for _ in range(E)]
    w["g_gamma"] = [o.pt_mul(o.G, g) for g in w["gamma"]]
    w["com"] = [g18.phase1_broadcast(g, b) for g, b in zip(w["g_gamma"], w["blind"])]
    w["s_i"] = [g18.phase5_local_sig(k, m, R, s) for k, m, R, s in zip(w["k"], w["m"], w["R"], w["sigma"])]
    for key in ("l", "rho", "blind5", "heg_s1", "heg_s2", "dlog_nonce", "blind2"):
        w[key] = [rng.randrange(1, Q) for _ in range(E)]
    return w


def _gg18_in(w, keys):
    return {k: (P(w[k]) if k in ("R", "y", "g_gamma") else L(w[k], 8)) for k in keys}


def _gg18_phase4(W, n):
    w = _gg18_world(n)
    inp = _gg18_in(w, ("delta_inv", "g_gamma", "blind", "com"))
    pk = [w["g_gamma"][u // PARTIES * PARTIES + j] for u in range(n * PARTIES) for j in range(PARTIES)]
    inp["b_proof_pk"] = P(pk)
    if n > 1:
        inp["com"] = tamper(inp["com"], n * PARTIES)                   # sessions with a commitment that does not reopen
    return inp, {"parties": PARTIES, "sessions": n}


def _gg18_phase4_check(W, i, s, x):
    u0 = s // PARTIES * PARTIES
    R = g18.phase4(row_int(i["delta_inv"], s), [row_pt(i["b_proof_pk"], s * PARTIES + j) for j in range(PARTIES)],
                   [(row_int(i["blind"], u0 + j), row_pt(i["g_gamma"], u0 + j)) for j in range(PARTIES)], [row_int(i["com"], u0 + j) for j in range(PARTIES)])
    return (x["status"][s, 0] == 0 and row_pt(x["R"], s) == R) if R is not None else x["status"][s, 0] == 2


GG18E = "sessions * parties"
spec("gg18_phase4_batch", [I("parties"), In("delta_inv", 8, GG18E), In("b_proof_pk", 16, GG18E + " * parties"), In("g_gamma", 16, GG18E), In("blind", 8, GG18E),
                           In("com", 8, GG18E), Out("R", 16, GG18E), Out("status", 1, GG18E, "u8"), Z("sessions")], check=_gg18_phase4_check)(_gg18_phase4)


@spec("gg18_local_sig_batch", [In("message", 8), In("R", 16), In("k_i", 8), In("sigma_i", 8), Out("s_i", 8), Z("count")],
      check=lambda W, i, s, x: row_int(x["s_i"], s) == g18.phase5_local_sig(row_int(i["k_i"], s), row_int(i["message"], s), row_pt(i["R"], s), row_int(i["sigma_i"], s)))
def _gg18_local(W, n):
    w = _gg18_world(n)
    inp = _gg18_in(w, ("m", "R", "k", "sigma"))
    return {"message": inp["m"][:n], "R": inp["R"][:n], "k_i": inp["k"][:n], "sigma_i": inp["sigma"][:n]}, {"count": n}


A5_IN = ("R", "s_i", "l_i", "rho_i", "blind", "heg_s1", "heg_s2", "dlog_nonce")
A5_OUT = [("com", 8), ("decom", 48), ("heg_proof", 48), ("dlog_proof", 40)]


def _gg18_5a_inputs(W, n, E):
    w = _gg18_world(n)
    src = {"R": "R", "s_i": "s_i", "l_i": "l", "rho_i": "rho", "blind": "blind5", "heg_s1": "heg_s1", "heg_s2": "heg_s2", "dlog_nonce": "dlog_nonce"}
    return {k: (P(w[v][:E]) if k == "R" else L(w[v][:E], 8)) for k, v in src.items()}


def _gg18_5a_check(W, i, s, x):
    a = g18.phase5a(*(row_int(i[k], s) for k in ("s_i", "l_i", "rho_i")), row_pt(i["R"], s), *(row_int(i[k], s) for k in ("blind", "heg_s1", "heg_s2", "dlog_nonce")))
    return x["status"][s, 0] == 0 and row_int(x["com"], s) == a.com and row_int(x["decom"], s) == pack(a.V) | pack(a.A) << 512 | pack(a.B) << 1024 and \
        _heg_pf(x["heg_proof"], s) == a.heg and _dlog_pf(x["dlog_proof"], s) == a.dlog


@spec("gg18_phase5a_batch", [In(k, 16 if k == "R" else 8) for k in A5_IN] + [Out(k, w) for k, w in A5_OUT] + [Out("status", 1, dt="u8"), Z("count")],
      check=_gg18_5a_check)
def _gg18_5a(W, n):
    return _gg18_5a_inputs(W, n, n), {"count": n}


C5_IN = [("R", 16), ("y", 16), ("message", 8), ("rho_i", 8), ("l_i", 8), ("blind2", 8), ("com", 8), ("decom", 48), ("blind", 8), ("heg_proof", 48), ("dlog_proof", 40)]


def _gg18_5c_inputs(W, n):
    w, E = _gg18_world(n), n * PARTIES
    a5_in = _gg18_5a_inputs(W, n, E)
    a5 = W.host("gg18_phase5a_batch", a5_in, {"count": E})
    inp = {"R": a5_in["R"], "y": P(w["y"]), "message": L(w["m"], 8), "rho_i": a5_in["rho_i"], "l_i": a5_in["l_i"], "blind2": L(w["blind2"], 8),
           "blind": a5_in["blind"]}
    inp.update({k: a5[k] for k, _ in A5_OUT})
    return inp, {"parties": PARTIES, "sessions": n}


def _gg18_5c(W, n):
    inp, sc = _gg18_5c_inputs(W, n)
    if n > 1:
        inp["heg_proof"] = tamper(inp["heg_proof"], n * PARTIES, 40)   # a signer whose ElGamal proof fails: its peers answer InvalidCom
    return inp, sc


spec("gg18_phase5c_batch", [I("parties")] + [In(k, w, GG18E) for k, w in C5_IN] + [Out("com2", 8, GG18E), Out("decom2", 32, GG18E),
                                                                                  Out("status", 1, GG18E, "u8"), Z("sessions")])(_gg18_5c)


def _gg18_5d(W, n):
    inp, sc = _gg18_5c_inputs(W, n)
    c5 = W.host("gg18_phase5c_batch", inp, sc)
    return {"decom2": c5["decom2"], "blind2": inp["blind2"], "com2": tamper(c5["com2"], n * PARTIES) if n > 1 else c5["com2"], "decom": inp["decom"]}, sc


spec("gg18_phase5d_batch", [I("parties"), In("decom2", 32, GG18E), In("blind2", 8, GG18E), In("com2", 8, GG18E), In("decom", 48, GG18E),
                            Out("status", 1, GG18E, "u8"), Z("sessions")])(_gg18_5d)


def _gg18_out_check(W, i, s, x):
    u0 = s // PARTIES * PARTIES
    code, sig = g18.output_signature(row_pt(i["R"], s), row_pt(i["y"], s), row_int(i["message"], s), [row_int(i["s_i"], u0 + j) for j in range(PARTIES)])
    return int(x["status"][s, 0]) == code and (sig is None or (row_int(x["sig_r"], s), row_int(x["sig_s"], s), int(x["recid"][s, 0])) == sig)


def _gg18_out(W, n):
    w = _gg18_world(n)
    inp = {"R": P(w["R"]), "y": P(w["y"]), "message": L(w["m"], 8), "s_i": L(w["s_i"], 8)}
    if n > 1:
        inp["s_i"] = tamper(inp["s_i"], n * PARTIES)
    return inp, {"parties": PARTIES, "sessions": n}


spec("gg18_output_signature_batch", [I("parties"), In("R", 16, GG18E), In("y", 16, GG18E), In("message", 8, GG18E), In("s_i", 8, GG18E),
                                     Out("sig_r", 8, GG18E), Out("sig_s", 8, GG18E), Out("recid", 1, GG18E, "u8"), Out("status", 1, GG18E, "u8"), Z("sessions")],
     check=_gg18_out_check)(_gg18_out)


# ------------------------------------------------------------------------------------------------ GG20 offline / online, sampler
def _sessions(W, n):
    rng = W.rng("sessions", n)
    pairs = [(0, 1), (0, 2), (1, 2), (1, 0), (2, 0), (2, 1)]
    s = [(rng.randrange(2), *rng.choice(pairs)) for _ in range(n)]
    s[-1] = (1, 0, 2)                                                  # an edge key set, and a non-zero last word
    return np.array(s, np.uint32)


def _rnd(W, sess):
    n = sess.shape[0]
    return W.host("gg20_sample_randomness", {"sessions": sess, "seed": _seed_arr()}, {"n_sessions": n, "first_unit": 0})["rnd"]


_seed_arr = lambda: np.frombuffer(SEED, "<u4").copy()


def _keysets_of(W):
    return [W.keys[:3], W.keys[3:]]


def _oracle_units(W, sess, s):
    k, a, b = sess[s].tolist()
    ks = _keysets_of(W)[k]
    keys, s_l = [ks[a], ks[b]], [a + 1, b + 1]
    units = [ss.sample_unit_seeded(SEED, 2 * s + p, keys, s_l, p) for p in range(2)]
    return keys, s_l, units


def _sample_rnd_check(W, i, s, x):
    from mpecdsa_b200 import gg20
    _, _, units = _oracle_units(W, i["sessions"], s)
    return np.array_equal(x["rnd"][2 * s:2 * s + 2], gg20.pack_randomness(units)) and not x["status"][2 * s:2 * s + 2].any()


@spec("gg20_sample_randomness", [KS, In("sessions", 3, "n_sessions"), Z("n_sessions"), HOSTBUF("seed"), U64("first_unit"), Out("rnd", 1408, "2 * n_sessions"),
                                 Out("status", 1, "2 * n_sessions", "u8")], check=_sample_rnd_check)
def _sample_rnd(W, n):
    return {"sessions": _sessions(W, n), "seed": _seed_arr()}, {"n_sessions": n, "first_unit": 0}


def _offline_check(W, i, s, x):
    keys, s_l, units = _oracle_units(W, i["sessions"], s)
    ref = o.offline_session(keys, s_l, units)
    return all(x["status"][2 * s + p, 0] == 0 and int.from_bytes(x["digest"][2 * s + p].tobytes(), "little").to_bytes(32, "big") == ref[p].transcript and
               row_int(x["sigma"], 2 * s + p) == ref[p].sigma_i and row_pt(x["R"], 2 * s + p) == ref[p].R for p in range(2))


OFF_OUT = [Out("status", 1, "2 * n_sessions", "u8"), Out("R", 16, "2 * n_sessions"), Out("sigma", 8, "2 * n_sessions"), Out("t_vec", 32, "2 * n_sessions"),
           Out("digest", 8, "2 * n_sessions")]


@spec("gg20_offline_batch", [KS, In("sessions", 3, "n_sessions"), Z("n_sessions"), In("rnd", 1408, "2 * n_sessions")] + OFF_OUT, check=_offline_check)
def _offline(W, n):
    sess = _sessions(W, n)
    return {"sessions": sess, "rnd": _rnd(W, sess)}, {"n_sessions": n}


def _records_check(W, i, s, x):
    off = W.host("gg20_offline_batch", {"sessions": i["sessions"][s:s + 1], "rnd": i["rnd"][2 * s:2 * s + 2]}, {"n_sessions": 1})
    rec = x["all_records"][2 * s:2 * s + 2]
    be = lambda a: np.ascontiguousarray(a[:, ::-1]).astype(">u4").view(np.uint8).reshape(2, -1)
    return not rec[:, 0].any() and np.array_equal(rec[:, 164:196], be(off["digest"])) and np.array_equal(rec[:, 66:98], be(i["rnd"][2 * s:2 * s + 2, 8:16]))


@spec("gg20_offline_records", [KS, NULL, In("sessions", 3, "n_sessions"), Z("n_sessions"), In("rnd", 1408, "2 * n_sessions"),
                               Out("all_records", 256, "2 * n_sessions", "u8")], check=_records_check)
def _records(W, n):
    return _offline(W, n)


def _sign_inputs(W, n):
    inp, sc = _offline(W, n)
    off = W.host("gg20_offline_batch", inp, sc)
    m = [W.rng("msg", n).getrandbits(256) for _ in range(n)]
    m[-1] = (1 << 256) - 1
    return {"sessions": inp["sessions"], "message": L(m, 8), "R": off["R"], "sigma": off["sigma"], "k": np.ascontiguousarray(inp["rnd"][:, 8:16])}, sc


def _sign_check(W, i, s, x):
    R = row_pt(i["R"], 2 * s)
    m = row_int(i["message"], s) % Q
    si = [o.local_sig(row_int(i["k"], 2 * s + p), m, R, row_int(i["sigma"], 2 * s + p)) for p in range(2)]
    r, sv, rec = o.output_signature(R, si)
    y = _keysets_of(W)[int(i["sessions"][s, 0])][0].y_sum_s
    return ints(x["s_i"][2 * s:2 * s + 2]) == si and (row_int(x["sig_r"], s), row_int(x["sig_s"], s), int(x["recid"][s, 0])) == (r, sv, rec) and \
        (x["status"][s, 0] == 0) == o.ecdsa_verify(r, sv, y, m)


@spec("gg20_sign_batch", [KS, In("sessions", 3, "n_sessions"), Z("n_sessions"), In("message", 8, "n_sessions"), In("R", 16, "2 * n_sessions"),
                          In("sigma", 8, "2 * n_sessions"), In("k", 8, "2 * n_sessions"), Out("s_i", 8, "2 * n_sessions"), Out("sig_r", 8, "n_sessions"),
                          Out("sig_s", 8, "n_sessions"), Out("recid", 1, "n_sessions", "u8"), Out("status", 1, "n_sessions", "u8")], check=_sign_check)
def _sign(W, n):
    return _sign_inputs(W, n)


def _sample_check(W, i, s, x):
    v, ok, _ = ss.sample(SEED, 7, 1000 + s, "below", row_int(i["bound"], int(i["bound_idx"][s])))
    return (row_int(x["out"], s), int(x["status"][s, 0])) == (v, 0 if ok else 13)


@spec("sample_batch", [HOSTBUF("seed"), U64("first_id"), U32("stream"), I("kind"), I("bits"), In("bound", "limbs", "n_bound or count"), In("bound_idx", 1),
                       Z("n_bound"), I("limbs"), Out("out", "limbs"), Out("status", 1, dt="u8"), Z("count")], check=_sample_check)
def _sample(W, n):
    rows = W.rows_for(n)
    return {"seed": _seed_arr(), "bound": L([W.N(r) for r in range(6)], 64), "bound_idx": np.array(rows, np.uint32)}, \
        {"first_id": 1000, "stream": 7, "kind": 1, "bits": 0, "n_bound": 6, "limbs": 64, "count": n}


# ------------------------------------------------------------------------------------------------ running one call
def _nbytes(a, sc):
    rows, width = _shape(a, sc)
    return rows * width * np.dtype(DT[a[2]]).itemsize


class _Buf:
    """One caller buffer between two GUARD-byte guards: numpy for HOST, a CUDA tensor for DEVICE; data 16-byte aligned."""

    def __init__(self, data: bytes, nb: int, mem, fill):
        self.nb, self.mem = nb, mem
        raw = bytearray([FILL_GUARD]) * (2 * GUARD + nb + 16)
        if mem == HOST:
            self.arr = np.frombuffer(raw, np.uint8).copy()
            self.off = GUARD + (-(self.arr.ctypes.data + GUARD)) % 16
        else:
            self.off = GUARD
        body = data if data is not None else bytes([fill]) * nb
        raw[self.off:self.off + nb] = body
        if mem == HOST:
            self.arr[:] = np.frombuffer(bytes(raw), np.uint8)
            self.ptr = self.arr.ctypes.data + self.off
        else:
            import torch
            self.arr = torch.frombuffer(bytearray(raw), dtype=torch.uint8).to("cuda", non_blocking=False)
            self.ptr = self.arr.data_ptr() + self.off
        assert self.ptr % 16 == 0
        self.before = bytes(raw)

    def now(self) -> bytes:
        return self.arr.tobytes() if self.mem == HOST else bytes(self.arr.cpu().numpy().tobytes())

    def data(self, b: bytes) -> bytes:
        return b[self.off:self.off + self.nb]

    def guards_ok(self, b: bytes) -> bool:
        return b[:self.off] == self.before[:self.off] and b[self.off + self.nb:] == self.before[self.off + self.nb:]


def _args(lib, ctx, ksh, sp, inp, sc, mem, guard=True, hold=None):
    """ctypes arguments of one call; buffers stay alive in `hold` (name -> _Buf or numpy array)"""
    hold = {} if hold is None else hold
    args = [ctx]                                                     # a c_void_p
    for a in sp.args:
        k = a[0]
        if k == "ks":
            args.append(ctypes.c_void_p(ksh))
        elif k == "null":
            args.append(ctypes.c_void_p(None))
        elif k == "int":
            args.append(ctypes.c_int(sc[a[1]]))
        elif k == "size":
            args.append(ctypes.c_size_t(sc[a[1]]))
        elif k == "u64":
            args.append(ctypes.c_uint64(sc[a[1]]))
        elif k == "u32":
            args.append(ctypes.c_uint32(sc[a[1]]))
        elif k == "host":
            hold[a[1]] = np.ascontiguousarray(inp[a[1]])
            args.append(ctypes.c_void_p(hold[a[1]].ctypes.data))
        else:
            name, nb = a[1], _nbytes(a, sc)
            if (k == "in" and inp.get(name) is None) or (k == "out" and name in sc.get("_null", ())):
                args.append(ctypes.c_void_p(None))
                continue
            data = None
            if k == "in":
                arr = np.ascontiguousarray(inp[name], dtype=DT[a[2]])
                rows, width = _shape(a, sc)
                assert arr.size == rows * width, (sp.id, name, arr.shape, rows, width)     # the builder agrees with the documented slot
                data = arr.tobytes()
            if not guard and mem == HOST:
                hold[name] = np.frombuffer(data, np.uint8).copy() if data is not None else np.full(max(nb, 1), FILL_OUT, np.uint8)
                args.append(ctypes.c_void_p(hold[name].ctypes.data))
            else:
                hold[name] = _Buf(data, nb, mem, FILL_OUT)
                args.append(ctypes.c_void_p(hold[name].ptr))
    args.append(ctypes.c_int(mem))
    return args, hold


def _outs(sp, sc, hold, snap=None):
    res = {}
    for a in sp.buffers("out"):
        if a[1] not in hold:
            continue
        rows, width = _shape(a, sc)
        h = hold[a[1]]
        b = h.data(snap[a[1]]) if isinstance(h, _Buf) else h[:_nbytes(a, sc)].tobytes()
        res[a[1]] = np.frombuffer(b, DT[a[2]]).reshape(rows, width).copy()
    return res


def _call(lib, ctx, ksh, sp, inp, sc, mem, guard=True):
    args, hold = _args(lib, ctx, ksh, sp, inp, sc, mem, guard)
    rc = getattr(lib, sp.fn)(*args)
    return rc, _outs(sp, sc, hold, {k: v.now() for k, v in hold.items() if isinstance(v, _Buf)})


def _guarded_run(eng, ksh, sp, inp, sc, mem, stream=None):
    """one call with every buffer guarded; -> (rc, outputs, list of problems: touched guards or changed inputs)"""
    import torch
    ctx_stream = torch.cuda.stream(stream) if stream is not None else _Null()
    with ctx_stream:
        args, hold = _args(eng.lib, eng._ctx, ksh, sp, inp, sc, mem)
        if mem == DEVICE:
            torch.cuda.current_stream().synchronize()                   # the buffers are in place before the library's stream reads them
        rc = getattr(eng.lib, sp.fn)(*args)
    if stream is not None:
        torch.cuda.current_stream().wait_stream(stream)
    snap = {k: v.now() for k, v in hold.items() if isinstance(v, _Buf)}
    bad = []
    for a in sp.buffers():
        h = hold.get(a[1])
        if not isinstance(h, _Buf):
            continue
        if not h.guards_ok(snap[a[1]]):
            bad.append(f"{a[1]}: guard touched")
        if a[0] == "in" and snap[a[1]] != h.before:
            bad.append(f"{a[1]}: input changed")
    return rc, _outs(sp, sc, hold, snap), bad


class _Null:
    def __enter__(self):
        return self

    def __exit__(self, *a):
        return False


# ------------------------------------------------------------------------------------------------ coverage (no GPU)
def header_entry_points(path=HEADER):
    src = open(path).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return {m.group(1) for m in re.finditer(r"\bint\s+(tecdsa_\w+)\s*\(([^;]*?)\bint\s+mem\s*\)\s*;", src, flags=re.S)}


def test_spec_table_covers_every_mem_entry_point():
    """every prototype of the header that ends in `int mem)` has an entry (and every entry names one), so a new entry point cannot
    skip the DEVICE/HOST comparison; each entry's buffers are named once and the table's argument count matches the prototype's"""
    want = header_entry_points()
    assert len(want) >= 67
    have = {s.fn for s in SPECS}
    assert have == want, {"missing": sorted(want - have), "unknown": sorted(have - want)}
    src = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    for s in SPECS:
        proto = re.search(r"\bint\s+" + s.fn + r"\s*\(([^;]*?)\)\s*;", src, flags=re.S).group(1)
        n_params = len([p for p in proto.split(",") if p.strip()])
        assert n_params == len(s.args) + 2, (s.id, n_params, len(s.args))          # + ctx, mem
        names = [a[1] for a in s.buffers()]
        assert len(names) == len(set(names)), s.id
        roles = {a[1]: a[0] for a in s.buffers()}
        for p in proto.split(","):                                                    # const pointers are inputs, the rest outputs
            m = re.match(r"\s*(const\s+)?\w+\s*\*\s*(\w+)", p)
            if m and m.group(2) in roles:
                assert roles[m.group(2)] == ("in" if m.group(1) else "out"), (s.id, m.group(2))


def test_header_parser_sees_a_new_prototype(tmp_path):
    """the coverage test above fails for an entry point the table does not know"""
    src = open(HEADER).read()
    extra = "int tecdsa_made_up_batch(tecdsa_ctx* ctx, const uint32_t* a,\n                          uint32_t* out, size_t count, int mem);\n"
    path = tmp_path / "h.h"
    path.write_text(src.replace("#ifdef __cplusplus\n}", extra + "#ifdef __cplusplus\n}", 1))
    assert header_entry_points(str(path)) - {s.fn for s in SPECS} == {"tecdsa_made_up_batch"}


# ------------------------------------------------------------------------------------------------ GPU fixtures
@pytest.fixture(scope="module")
def keys(keyset):
    edge = fixtures.load_edge_keysets()
    pick = next(ks for ks in edge if any((lk.dk.p * lk.dk.q).bit_length() == 2047 for lk in ks))
    return list(keyset) + list(pick)


@pytest.fixture(scope="module")
def world(engine, keys):
    from mpecdsa_b200 import gg20
    ks = gg20.KeySets(engine, [keys[:3], keys[3:]])
    yield World(engine, ks.handle.value, keys)
    ks.free()


@pytest.fixture(scope="module")
def private(pkg, keys):
    """a second context on a private stream, with its own upload of the key sets"""
    import torch
    from mpecdsa_b200 import gg20
    s = torch.cuda.Stream()
    eng = pkg.Engine(0, stream=s.cuda_stream)
    ks = gg20.KeySets(eng, [keys[:3], keys[3:]])
    yield eng, ks.handle.value, s
    ks.free()
    eng.close()


_INPUTS = {}


def _inputs(W, sp, n):
    key = (sp.id, n)
    if key not in _INPUTS:
        _INPUTS[key] = sp.build(W, n)
    return _INPUTS[key]


def _count_of(sp, sc):
    return sc.get("count", sc.get("n_sessions", sc.get("sessions")))


# ------------------------------------------------------------------------------------------------ GPU: every entry point, three runs
@pytest.mark.gpu
@pytest.mark.parametrize("n", COUNTS)
@pytest.mark.parametrize("sp", SPECS, ids=lambda s: s.id)
def test_device_buffers_equal_host_buffers(engine, world, private, sp, n):
    inp, sc = _inputs(world, sp, n)
    peng, pks, pstream = private
    rc_h, out_h, bad_h = _guarded_run(engine, world.ksh, sp, inp, sc, HOST)
    assert rc_h == 0, (sp.id, engine.lib.tecdsa_last_error())
    assert not bad_h, ("HOST", bad_h)
    rc_d, out_d, bad_d = _guarded_run(engine, world.ksh, sp, inp, sc, DEVICE)
    rc_p, out_p, bad_p = _guarded_run(peng, pks, sp, inp, sc, DEVICE, pstream)
    assert not bad_d and not bad_p, ("DEVICE", bad_d, "private stream", bad_p)
    if sp.host_only:                                                   # refused before anything is touched
        assert rc_d == rc_p == E_UNSUPPORTED
        assert all((v == FILL_OUT).all() for v in list(out_d.values()) + list(out_p.values()))
        return
    assert rc_d == rc_p == 0
    for name in out_h:
        assert out_h[name].tobytes() == out_d[name].tobytes(), (name, "session context")
        assert out_h[name].tobytes() == out_p[name].tobytes(), (name, "private stream")
    # the last element is valid (untampered, in range): its status is OK and its ok flag set — a verifier input made by a prover whose
    # inputs were staged wrongly is rejected here rather than agreeing with an equally rejecting DEVICE run
    for name, want in (("status", 0), ("ok", 1)):
        if name in out_h:
            assert int(out_h[name][-1, 0]) == want, (name, out_h[name][-1, 0])
    status = out_h.get("status")
    if status is not None and n > 3 and sp.id.endswith(("verify_batch", "message_b_batch", "get_alpha_batch", "message2_batch", "finalize_batch")):
        assert len(set(status[:, 0].tolist())) > 1, "a verifier batch mixes accepted and rejected elements"
    if sp.check is not None:                                           # the first and the last element against the oracle
        m = sc["sessions"] * sc["parties"] if "sessions" in sc else _count_of(sp, sc)
        for s in (0, m - 1):
            assert sp.check(world, inp, s, out_h), (sp.id, "element", s)


# ------------------------------------------------------------------------------------------------ GPU: chains of DEVICE calls, one sync
def _find(fn, variant=""):
    return next(s for s in SPECS if s.fn == "tecdsa_" + fn and s.id.endswith(variant))


class _Dev:
    """DEVICE calls on one context: every buffer is a CUDA tensor made on the context's stream, and outputs are fed to later
    calls as they are, with no sync in between"""

    def __init__(self, eng, ksh, stream):
        self.eng, self.ksh, self.stream = eng, ksh, stream
        self.keep = []

    def call(self, fn, inp, sc, variant=""):
        """inp values: numpy arrays (uploaded here) or CUDA tensors from earlier calls; -> dict of output tensors (raw bytes)"""
        import torch
        sp = _find(fn, variant)
        args, outs = [self.eng._ctx], {}
        with torch.cuda.stream(self.stream):
            for a in sp.args:
                k = a[0]
                if k == "ks":
                    args.append(ctypes.c_void_p(self.ksh))
                elif k == "null":
                    args.append(ctypes.c_void_p(None))
                elif k in ("int", "size", "u64", "u32"):
                    args.append({"int": ctypes.c_int, "size": ctypes.c_size_t, "u64": ctypes.c_uint64, "u32": ctypes.c_uint32}[k](sc[a[1]]))
                elif k == "host":
                    h = np.ascontiguousarray(inp[a[1]])
                    self.keep.append(h)
                    args.append(ctypes.c_void_p(h.ctypes.data))
                elif k == "in":
                    v = inp.get(a[1])
                    if v is None:
                        args.append(ctypes.c_void_p(None))
                        continue
                    if not isinstance(v, torch.Tensor):
                        v = torch.from_numpy(np.ascontiguousarray(v, DT[a[2]]).view(np.uint8).reshape(-1).copy()).to("cuda")
                    assert v.numel() * v.element_size() == _nbytes(a, sc), (fn, a[1])
                    self.keep.append(v)
                    args.append(ctypes.c_void_p(v.data_ptr()))
                elif a[1] in sc.get("_null", ()):
                    args.append(ctypes.c_void_p(None))
                else:
                    outs[a[1]] = torch.empty(_nbytes(a, sc), dtype=torch.uint8, device="cuda")
                    args.append(ctypes.c_void_p(outs[a[1]].data_ptr()))
            args.append(ctypes.c_int(DEVICE))
            rc = getattr(self.eng.lib, sp.fn)(*args)
        assert rc == 0, (fn, self.eng.lib.tecdsa_last_error())
        return outs


def _cols(a, width, lo, w):
    """limbs [lo, lo + w) of every `width`-limb row: of a numpy array, or (on the current stream) of a CUDA tensor of raw bytes"""
    import torch
    if isinstance(a, torch.Tensor):
        return a.view(torch.int32).view(-1, width)[:, lo:lo + w].contiguous().view(torch.uint8).reshape(-1)
    return np.ascontiguousarray(a.reshape(a.shape[0], width)[:, lo:lo + w])


def _run_chains(W, chains):
    """chains: list of (_Dev, steps), steps = [(fn, variant, mk)], mk(previous outputs of its chain) -> (inputs, scalars).  Every chain
    runs once on HOST through the session context (each output read back) and once on DEVICE through its _Dev (outputs passed on as
    tensors), the DEVICE calls of all chains interleaved step by step and nothing read before the end.  Asserts byte equality;
    -> the HOST outputs of every chain."""
    import torch
    host = [[] for _ in chains]
    dev = [[] for _ in chains]
    for step in range(max(len(s) for _, s in chains)):
        for c, (d, steps) in enumerate(chains):
            if step >= len(steps):
                continue
            fn, variant, mk = steps[step]
            inp, sc = mk(host[c])
            host[c].append(W.host(fn, inp, sc, variant))
            with torch.cuda.stream(d.stream):
                dinp, _ = mk(dev[c])
            dev[c].append(d.call(fn, dinp, sc, variant))
    for c, (d, steps) in enumerate(chains):
        torch.cuda.current_stream().wait_stream(d.stream)
    for c in range(len(chains)):
        for i, (h, g) in enumerate(zip(host[c], dev[c])):
            assert set(h) >= set(g)
            for k in g:
                assert h[k].tobytes() == g[k].cpu().numpy().tobytes(), (c, i, chains[c][1][i][0], k)
    return host


def _paillier_chain(W, n, variant, tag):
    rng, rows = W.rng(tag, n), W.rows_for(n)
    key = {"n": L([W.N(r) for r in range(6)], 64), "key_idx": np.array(rows, np.uint32)} if variant == "idx" else \
        {"n": L([W.N(r) for r in rows], 64), "key_idx": None}
    sc = {"n_keys": 6 if variant == "idx" else 0, "count": n}
    m, m2 = ([rng.randrange(W.N(r) // 2) for r in rows] for _ in range(2))
    r = [W.unit(rng, W.N(x)) for x in rows]
    k = [rng.getrandbits(256) for _ in rows]
    steps = [
        ("paillier_encrypt_batch", variant, lambda p: (dict(key, m=L(m, 64), r=L(r, 64)), sc)),
        ("paillier_encrypt_batch", variant, lambda p: (dict(key, m=L(m2, 64), r=L(r, 64)), sc)),
        ("paillier_mul_batch", variant, lambda p: (dict(key, c=p[0]["c"], k=L(k, 8)), dict(sc, k_limbs=8))),
        ("paillier_add_batch", variant, lambda p: (dict(key, c1=p[2]["out"], c2=p[1]["c"]), sc)),
        ("paillier_decrypt_batch", "", lambda p: ({"key_row": np.array(rows, np.uint32), "c": p[3]["out"]}, {"count": n})),
    ]
    want = [(m[i] * k[i] + m2[i]) % W.N(rows[i]) for i in range(n)]
    return steps, want


@pytest.mark.gpu
@pytest.mark.parametrize("variant", ["idx", "rows"])
def test_paillier_chain_on_a_private_stream(world, private, variant):
    """encrypt -> mul -> add -> decrypt, each DEVICE output the next call's input, with and without key_idx"""
    peng, pks, ps = private
    n = 65
    steps, want = _paillier_chain(world, n, variant, "pchain")
    host = _run_chains(world, [(_Dev(peng, pks, ps), steps)])[0]
    dec = ints(host[4]["m"])
    assert [dec[0], dec[-1]] == [want[0], want[-1]]


def _mta_chain(W, n, tag):
    inp_b, sc, inp_a = _mta_b_inputs(W, n, tag)
    tail = {k: inp_b[k] for k in ("b",) + tuple(k for k, _ in MTA_B_IN)}
    steps = [
        ("mta_message_a_batch", "", lambda p: (inp_a, sc)),
        ("mta_message_b_batch", "", lambda p: (dict(tail, ek_row=inp_a["ek_row"], st_rows=inp_a["st_rows"], c_a=p[0]["c"],
                                                     **{k: p[0][k] for k, _ in MTA_A_OUT}), sc)),
        ("mta_get_alpha_batch", "", lambda p: ({"dk_row": inp_a["ek_row"], "a": inp_a["a"], "c_b": p[1]["c_b"], "b_proof": p[1]["b_proof"],
                                                "beta_tag_proof": p[1]["beta_tag_proof"]}, {"count": n})),
    ]
    a, b, bt = ints(inp_a["a"]), ints(inp_b["b"]), ints(inp_b["beta_tag"])
    return steps, [(a[i] * b[i] + bt[i]) % Q for i in range(n)]


@pytest.mark.gpu
def test_mta_chain_on_a_private_stream(world, private):
    """message_a -> message_b -> get_alpha on DEVICE buffers"""
    peng, pks, ps = private
    n = 65
    steps, want = _mta_chain(world, n, "mta-chain")
    host = _run_chains(world, [(_Dev(peng, pks, ps), steps)])[0]
    assert not host[1]["status"].any() and not host[2]["status"].any()
    alpha = ints(host[2]["alpha"])
    assert [alpha[0], alpha[-1]] == [want[0], want[-1]]


@pytest.mark.gpu
def test_lindell17_chain_on_a_private_stream(world, private):
    """Lindell-2017 key generation and signing as DEVICE calls: party one's DLogProof and key commitment, party two's check of the
    proof, the Paillier encryption of x1, the four messages of the interactive PDL proof, both ephemeral-key messages and their
    checks, the partial signature, the signature and its verification against x1 x2 G"""
    peng, pks, ps = private
    n, W = 65, world
    rng, rows = W.rng("l17chain", n), W.rows_for(n)
    x1, x2, k1, k2 = (scalars(rng, n) for _ in range(4))
    nonces = [L(scalars(rng, n), 8) for _ in range(3)]
    blinds = [L(scalars(rng, n, (1 << 256) - 1), 8) for _ in range(4)]
    key = {"n": L([W.N(r) for r in range(6)], 64), "key_idx": np.array(rows, np.uint32)}
    sc, sck = {"count": n}, {"n_keys": 6, "count": n}
    rnd = L([W.unit(rng, W.N(v)) for v in rows], 64)
    msg = L([rng.getrandbits(256) for _ in rows], 8)
    a, b = L([rng.randrange(Q) for _ in rows], 8), L([rng.randrange(Q * Q) for _ in rows], 16)
    rho = L([rng.randrange(Q * Q) for _ in rows], 16)
    pk1 = lambda p: _cols(p[0]["proof"], 40, 0, 16)
    steps = [
        ("dlog_prove_batch", "", lambda p: ({"sk": L(x1, 8), "nonce": nonces[0]}, sc)),                                           # 0
        ("hash_commitment_batch", "", lambda p: ({"points": pk1(p), "blind": blinds[0]}, sc)),                                     # 1
        ("dlog_verify_batch", "", lambda p: ({"proof": p[0]["proof"]}, sc)),                                                       # 2
        ("paillier_encrypt_batch", "idx", lambda p: (dict(key, m=L(x1, 64), r=rnd), sck)),                                         # 3
        ("zkpdl_verifier_message1_batch", "", lambda p: (dict(key, ciphertext=p[3]["c"], Q=pk1(p), a=a, b=b, randomness=rnd, blindness=blinds[1]), sck)),
        ("zkpdl_prover_message1_batch", "", lambda p: ({"key_row": key["key_idx"], "c_tag": p[4]["c_tag"], "blindness": blinds[2]}, sc)),   # 5
        ("zkpdl_prover_message2_batch", "", lambda p: ({"x1": L(x1, 8), "alpha": p[5]["alpha"], "c_tag_tag": p[4]["c_tag_tag"], "a": a, "b": b,
                                                        "blindness": blinds[1]}, sc)),                                             # 6
        ("zkpdl_verifier_finalize_batch", "", lambda p: ({"c_hat": p[5]["c_hat"], "q_hat": p[5]["q_hat"], "blindness": blinds[2], "q_tag": p[4]["q_tag"]}, sc)),
        ("l17_eph_create_batch", "", lambda p: ({"secret_share": L(k1, 8), "nonce": nonces[1], "pk_blind": None, "zk_pok_blind": None},
                                                dict(sc, _null=("pk_commitment", "zk_pok_commitment")))),                         # 8: party one
        ("l17_eph_create_batch", "", lambda p: ({"secret_share": L(k2, 8), "nonce": nonces[2], "pk_blind": blinds[3], "zk_pok_blind": blinds[0]}, sc)),
        ("l17_eph_verify_batch", "", lambda p: ({"public_share": p[8]["public_share"], "c_point": p[8]["c_point"], "proof": p[8]["proof"]}, sc)),
        ("l17_eph_verify_batch", "", lambda p: ({k: p[9][k] for k in ("public_share", "c_point", "proof", "pk_commitment", "zk_pok_commitment")} |
                                                {"pk_blind": blinds[3], "zk_pok_blind": blinds[0]}, sc)),                         # 11
        ("l17_partial_sig_batch", "", lambda p: (dict(key, c_key=p[3]["c"], x2=L(x2, 8), k2=L(k2, 8), eph_other_public=p[8]["public_share"],
                                                      message=msg, rho=rho, randomness=rnd), sck)),                               # 12
        ("l17_sign_batch", "", lambda p: ({"key_row": key["key_idx"], "c3": p[12]["c3"], "k1": L(k1, 8), "eph_other_public": p[9]["public_share"]}, sc)),
        ("secp_mul_batch", "", lambda p: ({"points": pk1(p), "scalars": L(x2, 8)}, sc)),                                           # 14: x1 x2 G
        ("l17_verify_batch", "", lambda p: ({"sig_r": p[13]["sig_r"], "sig_s": p[13]["sig_s"], "pubkey": p[14]["out"], "message": msg}, sc)),
    ]
    host = _run_chains(W, [(_Dev(peng, pks, ps), steps)])[0]
    for i in (2, 4, 5, 6, 7, 10, 11, 12, 13, 15):
        assert not host[i]["status"].any(), (i, steps[i][0])


def _gg20_chain(W, n, seed_tag):
    sess = _sessions(W, n)
    m = [W.rng(seed_tag, n).getrandbits(256) for _ in range(n)]
    sc = {"n_sessions": n}
    steps = [
        ("gg20_sample_randomness", "", lambda p: ({"sessions": sess, "seed": _seed_arr()}, dict(sc, first_unit=0))),
        ("gg20_offline_batch", "", lambda p: ({"sessions": sess, "rnd": p[0]["rnd"]}, sc)),
        ("gg20_sign_batch", "", lambda p: ({"sessions": sess, "message": L(m, 8), "R": p[1]["R"], "sigma": p[1]["sigma"],
                                            "k": _cols(p[0]["rnd"], 1408, 8, 8)}, sc)),
        ("gg20_offline_records", "", lambda p: ({"sessions": sess, "rnd": p[0]["rnd"]}, sc)),
    ]
    return steps


@pytest.mark.gpu
def test_gg20_chain_on_a_private_stream(world, private):
    """sample_randomness -> offline_batch -> sign_batch, and offline_records with a NULL communicator, on DEVICE buffers"""
    peng, pks, ps = private
    n = 65
    host = _run_chains(world, [(_Dev(peng, pks, ps), _gg20_chain(world, n, "gg20chain"))])[0]
    assert not host[0]["status"].any() and not host[1]["status"].any() and not host[2]["status"].any()
    assert not host[3]["all_records"][:, 0].any()


@pytest.mark.gpu
def test_two_contexts_interleaved(world, private, pkg, keys):
    """two contexts on two private streams, DEVICE calls of different entry points alternating between them from one thread:
    each context's results equal its serial HOST results"""
    import torch
    from mpecdsa_b200 import gg20
    peng, pks, ps = private
    s2 = torch.cuda.Stream()
    eng2 = pkg.Engine(0, stream=s2.cuda_stream)
    ks2 = gg20.KeySets(eng2, [keys[:3], keys[3:]])
    try:
        n = 65
        a_steps, want = _paillier_chain(world, n, "idx", "two-a")
        b_steps, want_b = _mta_chain(world, n, "two-b")
        c_steps = _gg20_chain(world, n, "two-c")
        da, db = _Dev(peng, pks, ps), _Dev(eng2, ks2.handle.value, s2)
        host = _run_chains(world, [(da, a_steps), (db, b_steps), (da, c_steps), (db, a_steps[:3])])
        assert ints(host[0][4]["m"])[-1] == want[-1]
        assert ints(host[1][2]["alpha"])[-1] == want_b[-1]
    finally:
        torch.cuda.synchronize()
        ks2.free()
        eng2.close()
