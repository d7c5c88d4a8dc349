"""CPU: round 1's AliceProof u' = (s1 N + 1) * s^N * (c^-1)^e mod N^2 of the fused GG20 offline stage evaluated through the
CRT halves of the peer's key row (declared shortcut 12, DESIGN.md section 4), restated with Python integers stage by stage as
csrc/gg20.cu stages it and recombined by crt_combine (csrc/gg20_glue.cuh) compiled for the host:

  1. 1024-bit list:  TP = (s mod p)^(q mod (p-1)) mod p,  TQ likewise;
  2. p-adic list:    YP = TP^p * (cinv mod p^2)^e * (gs1 mod p^2) mod p^2,  YQ likewise;
  3. gg20_crt:       u' from (YP, YQ) in [0, N^2).

Every row of keys_t1n3.json and keys_edge.json, with s at the values where b^N mod p^2 could break (0, 1, p, q, N - 1, N,
N + p, 2^2048 - 1) and with a c^-1 operand that is at least N^2 (the p-adic lift reduces any operand up to 4096 bits)."""
import ctypes
import random

import numpy as np

from tests.golden import fixtures
from tests.test_glue_host import KEY_SIZE, I, L, P, h  # noqa: F401  (h: the host harness fixture)


def _rows():
    return [lk for ks in fixtures.load_all_keysets() + fixtures.load_edge_keysets() for lk in ks]


def _staged_halves(s, cinv, e, gs1, p, q):
    """(YP, YQ) as stages 1 and 2 compute them"""
    def half(a, b):
        t = pow(s % a, b % (a - 1), a)
        aa = a * a
        return pow(t, a, aa) * pow(cinv % aa, e, aa) * (gs1 % aa) % aa
    return half(p, q), half(q, p)


def test_peer_u_prime_through_crt_halves(h):
    rows = _rows()
    assert len(rows) == 33
    tabs = [np.zeros((len(rows), s), np.uint32) for s in KEY_SIZE]
    for r, lk in enumerate(rows):
        tabs[9][r] = L(lk.dk.p, 32); tabs[10][r] = L(lk.dk.q, 32)
    ptrs = (ctypes.c_void_p * len(tabs))(*[t.ctypes.data for t in tabs])
    h.h_key_setup(ptrs, len(rows))
    rng = random.Random(0x9EE2C27)
    out = np.zeros(128, np.uint32)
    for r, lk in enumerate(rows):
        p, q = lk.dk.p, lk.dk.q
        N = p * q
        NN = N * N
        assert q % (p - 1) != 0 and p % (q - 1) != 0             # so s = 0 mod p gives TP = 0, as 0^N = 0
        for s in (0, 1, p, q, N - 1, N, N + p, (1 << 2048) - 1):
            e = rng.getrandbits(256)
            gs1 = rng.getrandbits(28 * 32) * N + 1
            cinv = rng.randrange(NN)
            sn = pow(s, N, NN)
            for c in (cinv, cinv + ((1 << 4096) - 1 - cinv) // NN * NN):    # and the largest c + j N^2 below 2^4096
                want = sn * pow(c, e, NN) * gs1 % NN
                yp, yq = _staged_halves(s, c, e, gs1, p, q)
                h.h_crt_combine(P(out), ptrs, r, P(L(yp, 64)), P(L(yq, 64)))
                assert I(out) == want, (r, s == p, s == q, c >= NN)
