"""Sliding windows for the exponents that are per-key constants (csrc/recode.h) and the fold of (c^-1)^e into the Straus
jobs of the verifiers' N-th powers.

CPU: the recoding compiled for the host reproduces the exponent, with odd, non-overlapping digits below 2^SLIDE_BITS.
GPU: nadic_jobs_kernel runs a class on the recoded digits only in warps whose lane groups share the key row, and fixed
windows elsewhere; offline batches over 8 key sets, whose key-row runs are not multiples of a warp, match the C twin unit
by unit, both unsplit and split into two half-batches.  The per-launch profile shows the round-1 launch of the separate
(c^-1)^e jobs gone."""
import ctypes
import os
import random
import subprocess

import numpy as np
import pytest

import __graft_entry__ as entry

SLIDE_BITS = 6
SHIM = r'''
#include "recode.h"
extern "C" void h_slide_recode(uint8_t* digits, const uint32_t* e, int limbs) { tecdsa::slide_recode(digits, e, limbs); }
'''


@pytest.fixture(scope="module")
def rec(tmp_path_factory):
    d = tmp_path_factory.mktemp("recode")
    src, so = d / "shim.cpp", d / "librecode.so"
    src.write_text(SHIM)
    here = os.path.join(os.path.dirname(os.path.abspath(__file__)), "host_harness")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-I", here, "-I", entry.CSRC, "-shared", "-fPIC", "-o", str(so), str(src)])
    lib = ctypes.CDLL(str(so))
    lib.h_slide_recode.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int]

    def run(e, limbs):
        ea = np.frombuffer(e.to_bytes(4 * limbs, "little"), dtype=np.uint32).copy()
        out = np.full(32 * limbs, 0xAA, dtype=np.uint8)
        lib.h_slide_recode(out.ctypes.data, ea.ctypes.data, limbs)
        return out
    return run


def _exponents():
    rng = random.Random(0x5711DE)
    out = []
    for limbs in (32, 64):
        B = 32 * limbs
        out += [(0, limbs), (1, limbs), ((1 << B) - 1, limbs), (1 << (B - 1), limbs), ((1 << (B - 1)) - 1, limbs)]
        out += [(1 << k, limbs) for k in (0, 5, 6, 7, 31, 32, 63, B - 2)]
        out += [((1 << k) - 1, limbs) for k in (5, 6, 7, 12, 33, B - 3)]
        out += [((1 << (B - 1)) | 1, limbs), (0b100001 << (B - 6), limbs), (0b11 << (B - 2), limbs)]          # short top window
        out += [(63 << s, limbs) for s in (0, 1, B - 6)] + [(0b111111000001, limbs)]                         # the largest odd digit
        out += [(rng.getrandbits(B), limbs) for _ in range(24)] + [(rng.getrandbits(B) | 1 | (1 << (B - 1)), limbs) for _ in range(8)]
    return out


@pytest.mark.parametrize("e,limbs", _exponents())
def test_recoding_reproduces_the_exponent(rec, e, limbs):
    d = rec(e, limbs)
    assert sum(int(v) << b for b, v in enumerate(d)) == e
    pos = np.nonzero(d)[0]
    assert all(d[pos] & 1) and all(d[pos] < 1 << SLIDE_BITS)
    # a digit's window spans its bit length; the next digit up starts above it
    spans = [(int(b), int(b) + int(d[b]).bit_length()) for b in pos]
    assert all(hi <= lo2 for (_, hi), (lo2, _) in zip(spans, spans[1:]))
    # greedy from the top: the top digit starts at the exponent's top bit
    assert not e or spans[-1][1] == e.bit_length()


# ------------------------------------------------------------------------------------------------ GPU
def _twin_equal(res, tw):
    assert np.array_equal(res.status, tw.status)
    assert not tw.status.any()
    for f in ("R", "sigma", "t_vec", "digest"):
        assert np.array_equal(np.asarray(getattr(res, f)).reshape(len(tw.status), -1),
                              np.asarray(getattr(tw, f)).reshape(len(tw.status), -1)), f


@pytest.mark.gpu
@pytest.mark.parametrize("n_sessions,seed", [(61, 0x51DE01), (2053, 0x51DE02)])
def test_offline_over_eight_keysets_matches_twin_on_every_unit(engine, n_sessions, seed):
    """61 sessions: most warps of a class straddle key rows (fixed windows) next to warps on one row (sliding windows);
    2053 sessions: split into two unequal half-batches, each with its own instance orders."""
    from mpecdsa_b200 import gg20
    from oracle import twin
    from tests.golden import fixtures
    keysets = fixtures.load_all_keysets()
    sess, rnd = gg20.synthetic_batch(keysets, n_sessions, seed)
    rows = np.bincount(np.concatenate([sess[:, 0] * 3 + sess[:, 1], sess[:, 0] * 3 + sess[:, 2]]), minlength=24)
    assert (rows % 4 != 0).any() and (rows % 8 != 0).any()           # runs that end inside a warp of the N^2 and p^2 kernels
    ks = gg20.KeySets(engine, keysets)
    try:
        res = gg20.offline_batch(engine, ks, sess, rnd)
    finally:
        ks.free()
    _twin_equal(res, twin.offline_batch(twin.KeyTables(keysets), sess, rnd, os.cpu_count() or 1))


@pytest.mark.gpu
def test_folded_inverse_powers_are_gone(engine, pkg):
    """(c^-1)^e no longer runs as jobs of its own in round 1: one N^2 launch fewer per offline call, and its arena fields
    are gone; the own proof's (c^-1)^e of round 5 stays (its consumer has no base to pair it with)."""
    from mpecdsa_b200 import gg20
    from tests.golden import fixtures
    keysets = fixtures.load_all_keysets()
    sess, rnd = gg20.synthetic_batch(keysets, 24, 0x51DE03)
    ks = gg20.KeySets(engine, keysets)
    try:
        prof = engine.profile_step(lambda: gg20.offline_batch(engine, ks, sess, rnd))
        for name in ("CEI0", "CEI1", "CEI2", "VCEI1"):
            with pytest.raises(pkg.EngineError, match="unknown field"):
                gg20.debug_field(engine, name, 48)
        assert gg20.debug_field(engine, "VCEI0", 48).shape == (48, 128)
    finally:
        ks.free()
    nn = [v for k, v in prof.items() if k.startswith("nadic_jobs_kernel<64")]
    assert len(nn) == 1 and nn[0]["launches"] == 5, prof             # rounds 0, 1, 4 and two in round 5
