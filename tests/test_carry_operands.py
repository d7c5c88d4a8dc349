"""Coverage witness for the carry-stress operand families (tests/carry_operands.py): for every (K, TPI) the GPU carry tests
run, the families contain additions whose carry travels through 1, 2, ... TPI-1 consecutive all-ones lanes as group_carry
resolves it, and plain operands whose N-adic lift has zero low quotient lanes.  Uniform random operands reach neither, so
this shows the GPU tests exercise those paths rather than hoping they do."""
import random

import pytest

from tests import carry_operands as co

# (bits, TPI) of every lane-group instantiation tests/test_carry_stress_gpu.py drives: the modexp shapes set_tpi accepts,
# the job kernels of modmul / modinv (2048: 4 lanes, 4096: 8) and the N-adic kernels (K = 64: 8 or 4 lanes; K = 32: 4 or 2)
SHAPES = sorted({(1024, t) for t in (4, 8, 16)} | {(2048, t) for t in (4, 8, 16, 32)} | {(4096, t) for t in (8, 16, 32)}
                | {(1024, 2)})


def _pairs(bits, tpi, rng):
    """The operand pairs the kernels add: x + y (group_add_masked, rows_finish) and x - y = x + ~y + 1 (group_sub_masked)
    over the lane-aligned values, the structured values and the moduli with their boundary residues."""
    vals = co.structured(bits, tpi, rng)
    ms = co.moduli(bits, tpi, rng)
    for n in ms:
        vals += co.residues(n, bits)
    vals += ms + [1, 2]
    R = 1 << bits
    for x in vals:
        for y in vals:
            yield x, y, 0
            yield x, (R - 1) ^ y, 1


@pytest.mark.parametrize("bits,tpi", SHAPES)
def test_families_propagate_carries_through_every_run_length(bits, tpi):
    rng = random.Random(bits * 131 + tpi)
    K = bits // 32
    seen = set()
    for x, y, c in _pairs(bits, tpi, rng):
        seen.update(co.model_propagate_runs(x, y, K, tpi, c))
        if seen >= set(range(1, tpi)):
            break
    assert set(range(1, tpi)) <= seen, (bits, tpi, sorted(seen))


def test_uniform_operands_do_not_propagate():
    """the contrast the families exist for: 2000 uniform additions at 2048 bits / 4 lanes never run a carry through a lane"""
    rng = random.Random(5)
    K, tpi = 64, 4
    assert not any(co.model_propagate_runs(rng.getrandbits(2048), rng.getrandbits(2048), K, tpi) for _ in range(2000))


@pytest.mark.parametrize("K,tpi", [(64, 8), (64, 4), (32, 4), (32, 2)])
def test_lifts_with_zero_low_quotient_lanes(K, tpi):
    """Every lane count j = 1..TPI-1 of zero low quotient lanes occurs when the N-adic lift of the families' ciphertexts
    (multiples of 2^(32Lj) and the other lane-aligned values) runs modulo the families' odd N."""
    rng = random.Random(K * 7 + tpi)
    bits = 32 * K
    ns = co.moduli(bits, tpi, rng)
    cts = co.lane_values(2 * K, 2 * tpi, rng)            # 2K-limb ciphertexts: lane boundaries of both chunks
    seen = set()
    for n in ns:
        for c in cts:
            seen.update(co.nadic_zero_quotient_lanes(c, n, K, tpi))
    assert set(range(1, tpi)) <= seen, sorted(seen)


def test_rrandomb_runs_and_top_bit():
    rng = random.Random(1)
    for bits in (1, 2, 31, 32, 33, 2047, 2048, 4096):
        for top in (True, False, None):
            x = co.rrandomb(bits, rng, top)
            assert 0 <= x < 1 << bits
            if top is True:
                assert x >> (bits - 1) == 1
            if top is False:
                assert x >> (bits - 1) == 0 if bits > 0 else True
    # long runs: a 4096-bit value has far fewer bit flips than the ~2048 of a uniform one
    flips = [bin(x ^ (x >> 1)).count("1") for x in (co.rrandomb(4096, rng, True) for _ in range(20))]
    assert max(flips) < 200


def test_families_are_well_formed():
    rng = random.Random(2)
    for bits, tpi in ((1024, 4), (2048, 4), (2048, 32), (4096, 8)):
        R = 1 << bits
        ms = co.moduli(bits, tpi, rng)
        assert all(n & 1 and 1 < n < R for n in ms)
        assert any(R - n < 1 << 32 for n in ms)
        assert any(n & 0xFFFFFFFF == 1 for n in ms) and any(n & 0xFFFFFFFF == 0xFFFFFFFF for n in ms)
        assert any(n.bit_length() == bits - 1 for n in ms) and any(n.bit_length() <= bits - bits // tpi for n in ms)
        for n in ms:
            assert all(0 <= r < R for r in co.residues(n, bits))
            for a, b in co.product_pairs(n, rng):
                assert 0 <= a < R and 0 <= b < R
            assert {a * b % n for a, b in co.product_pairs(n, rng)} >= {0, 1, n - 1}
        assert all(0 <= v < R for v in co.lane_values(bits // 32, tpi, rng))
    for ebits in (32, 64, 96, 2048):
        es = co.exponents(ebits, rng)
        assert all(0 <= e < 1 << ebits for e in es) and (1 << ebits) - 1 in es
        assert (1 << 5) in es and (1 << 5) - 1 in es and (ebits <= 32 or 1 << 32 in es)
