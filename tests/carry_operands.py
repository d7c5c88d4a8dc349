"""Structured operands that drive the carry paths of the lane-group big-integer kernels.

A K-limb operand is spread over TPI lanes of L = K/TPI limbs each (csrc/bigint.cuh).  Uniformly random limbs almost never
make a lane all-ones after an in-lane addition (about 2^-(32 L) per lane), so the propagate path of group_carry, the second
carry word of rows_finish and the all-ones start of the N-adic product's second pass are out of their reach.  The families
here are built so that they are reached: GMP-style runs of ones and zeros (mpz_rrandomb), values whose lanes are all-ones or
all-zero at every lane boundary of a given (K, TPI), moduli just below R or just above 2^(bits-1), boundary residues and
exponents on window and limb boundaries.  Everything is deterministic given a random.Random.

model_propagate_runs and nadic_zero_quotient_lanes model, in plain integers, what the kernels do with such operands; the
CPU test tests/test_carry_operands.py uses them to show that the families reach the paths."""
from math import gcd

LIMB = 32
WINDOW_BITS = 5


def rrandomb(bits, rng, top=None):
    """A `bits`-bit value made of alternating runs of ones and zeros with random run lengths (GMP's mpz_rrandomb).
    top: True forces the top bit on, False forces it off, None leaves it to the runs."""
    if bits <= 0:
        return 0
    x, pos, bit = 0, bits, rng.getrandbits(1) if top is None else int(top)
    while pos > 0:
        run = min(pos, 1 + rng.getrandbits(rng.randrange(1, 11)))
        pos -= run
        if bit:
            x |= ((1 << run) - 1) << pos
        bit ^= 1
    if top is not None:
        x = x | (1 << (bits - 1)) if top else x & ((1 << (bits - 1)) - 1)
    return x


def lane_values(K, TPI, rng):
    """Values < R = 2^(32K) whose lanes (L = K/TPI limbs each) are all-ones or all-zero at each lane boundary j = 1..TPI-1:
    R - 2^(32Lj) (lanes j and up all-ones), 2^(32Lj) - 1 (lanes below j all-ones), each of them +- 1, one all-ones lane j
    with random lanes around it, and a nonzero multiple of 2^(32Lj) (zero low lanes)."""
    R, W = 1 << (LIMB * K), LIMB * K // TPI
    out = []
    for j in range(1, TPI):
        hi, lo = R - (1 << (W * j)), (1 << (W * j)) - 1
        out += [hi, hi - 1, hi + 1, lo, lo - 1, lo + 1]
        out.append(rng.getrandbits(LIMB * K) | (((1 << W) - 1) << (W * j)))
        out.append((rng.getrandbits(LIMB * K - W * j) | 1) << (W * j))
    out.append(rng.getrandbits(LIMB * K) | ((1 << W) - 1))          # lane 0 all-ones
    return out


def moduli(bits, TPI, rng):
    """Odd moduli of `bits` bits or fewer at the carry edges of a TPI-lane group (L = bits/32/TPI limbs per lane)."""
    R, W = 1 << bits, bits // TPI
    top = 1 << (bits - 1)
    ms = [R - 1, R - (1 << W) + 1, top + 1, top + (1 << W) - 1,
          R - (rng.getrandbits(31) | 1),                                                  # R - n < 2^32: ov = 1 in mont_mul
          (rng.getrandbits(bits) | top) & ~0xFFFFFFFF | 1,                                # n[0] = 1: n0inv = 2^32 - 1
          rng.getrandbits(bits) | top | 0xFFFFFFFF,                                        # n[0] = 2^32 - 1: n0inv = 1
          rrandomb(bits, rng, True) | 1, rrandomb(bits, rng, True) | 1,
          rrandomb(bits - 1, rng, True) | 1,                                              # 2047 bits at 2048
          rrandomb(bits - W, rng, True) | 1]                                              # a whole zero top lane
    return ms


def residues(n, bits):
    """Boundary residues of modulus n at width `bits` (all < 2^bits): n-1, n-2, (n-1)/2, (n+1)/2, R mod n, R - n."""
    R = 1 << bits
    return [n - 1, n - 2, (n - 1) // 2, (n + 1) // 2, R % n, R - n]


def product_pairs(n, rng):
    """(a, b) with a*b mod n equal to 0, 1 and n-1 (n odd > 2)."""
    out = [(0, rng.randrange(n)), (n, rng.randrange(n))]
    while True:
        a = rng.randrange(2, n)
        if gcd(a, n) == 1:
            break
    inv = pow(a, -1, n)
    out += [(a, inv), (inv, a), (a, (n - 1) * inv % n), (n - 1, n - 1), (n - 1, 1)]
    return out


def exponents(ebits, rng):
    """Exponents of at most `ebits` bits: all-ones, 2^j and 2^j - 1 on window (5-bit) and limb (32-bit) boundaries, runs."""
    # the first two window and limb boundaries, the middle limb and the last ones, each -1, +0, +1
    marks = {5, 10, 32, 64, LIMB * (ebits // LIMB // 2), ebits - ebits % WINDOW_BITS, ebits - ebits % LIMB, ebits - LIMB}
    js = sorted({j for m in marks for j in (m - 1, m, m + 1) if 0 < j < ebits} | {1, ebits - 1})
    out = [(1 << ebits) - 1, 0, 1]
    for j in js:
        out += [1 << j, (1 << j) - 1]
    out += [rrandomb(ebits, rng, True), rrandomb(ebits, rng, False), rrandomb(ebits, rng)]
    return out


def structured(bits, TPI, rng, count=6):
    """Mixed operands < 2^bits: lane-aligned values, runs with the top bit on, off or free, and the all-ones value."""
    out = lane_values(bits // LIMB, TPI, rng)
    out += [rrandomb(bits, rng, t) for t in (True, False, None) for _ in range(count // 3 or 1)]
    return out + [(1 << bits) - 1, 0, 1]


# ---------------------------------------------------------------------------------------------- models of the kernels
def lanes(x, K, TPI):
    """x as TPI lane values of 32K/TPI bits, lane 0 lowest."""
    W = LIMB * K // TPI
    return [(x >> (W * g)) & ((1 << W) - 1) for g in range(TPI)]


def model_propagate_runs(x, y, K, TPI, cin0=0):
    """The lane-group addition x + y + cin0 as group_carry resolves it: each lane adds its own L limbs (a carry out
    `generates`, an all-ones sum `propagates`), then the lookahead carries into each lane.  Returns the lengths of the runs
    of consecutive propagating lanes that a carry actually travels through (each such lane flips from all-ones to zero)."""
    W = LIMB * K // TPI
    xs, ys = lanes(x, K, TPI), lanes(y, K, TPI)
    s = [xs[g] + ys[g] + (cin0 if g == 0 else 0) for g in range(TPI)]
    gen = [v >> W for v in s]
    prop = [(v & ((1 << W) - 1)) == (1 << W) - 1 for v in s]
    runs, carry, run = [], 0, 0
    for g in range(TPI):
        if carry and prop[g]:
            run += 1
            continue
        if run:
            runs.append(run)
        run = 0
        carry = gen[g] or (carry and prop[g])
    if run:
        runs.append(run)
    return runs


def nadic_zero_quotient_lanes(c, N, K, TPI):
    """For a plain operand c < 2^(64K) lifted modulo N^2 by to_nadic: per K-limb chunk h, the number of low lanes of the
    first pass's Montgomery quotient m = -c_h * d0(R^(h+2) mod N^2) * N^-1 mod R that are zero.  The second pass of
    nadic_mul starts its accumulator at ~m + 1, so each such lane starts all-ones and the +1 has to ripple through it."""
    R, W = 1 << (LIMB * K), LIMB * K // TPI
    NN, ninv = N * N, pow(N, -1, R)
    out = []
    for h in range(2):
        ch = (c >> (LIMB * K * h)) & (R - 1)
        y0 = pow(R, h + 2, NN) % N
        m = (-ch * y0 * ninv) % R
        z = 0
        while z < TPI and (m >> (W * z)) & ((1 << W) - 1) == 0:
            z += 1
        out.append(z)
    return out
