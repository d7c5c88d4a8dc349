"""Generates tests/golden/keys_edge.json — GG20 (t=1, n=3) key sets at the edges of the key domain the reference accepts.

`keys_t1n3.json` comes from OpenSSL's RSA generator, which sets the top two bits of every prime: every N and N~ there has
exactly 2048 bits and p/q < 1.33.  The reference's keygen accepts any N and N~ of 2047 or 2048 bits
(gg_2020/party_i.rs:49-50, 287-290), so here each row is built to sit at one edge of that domain:

  unbalanced      p in [2^1024 - 2^1000, 2^1024), q the smallest 1023-bit values with pq >= 2^2046: p/q ~ 4, N just above 2^2046
  small_squares   p, q in [2^1023, 2^1023.5): N, p^2 and q^2 of 2047 bits
  min_n           p, q in [2^1023, 2^1023 + 2^1000): N just above 2^2046
  max_n           p, q in [2^1024 - 2^1000, 2^1024): N just below 2^2048
  ratio2          p in [2^1024 - 2^1000, 2^1024), q in [2^1023, 2^1023 + 2^1000): p/q ~ 2, both of 1024 bits
  balanced        p, q in [2^1023.5, 2^1024)
a `_swapped` suffix puts the larger factor in q (p < q).  N~ = p~ q~ has 2047 bits (p~, q~ in [2^1023, 2^1023.5)) or
2048 bits (p~, q~ in [2^1023.5, 2^1024)); "small_h1" draws h1 of 1200 bits, well below N~.  Each key set mixes 2047- and
2048-bit N~.  Feldman shares as in make_fixtures.py.

Primes come from a seeded `random.Random` and Miller-Rabin in plain Python, so a rerun writes a byte-identical file:
    python -m tests.golden.make_edge_keys
"""
import json
import os
import random
from math import gcd, isqrt

from oracle import gg20_oracle as o

HERE = os.path.dirname(os.path.abspath(__file__))
PATH = os.path.join(HERE, "keys_edge.json")

TOP, HALF, SLACK = 1 << 1024, 1 << 1023, 1 << 1000
MID = isqrt(1 << 2047) + 1                                   # 2^1023.5, rounded up: MID^2 > 2^2047
SMALL_PRIMES = [p for p in range(3, 2000) if all(p % d for d in range(2, isqrt(p) + 1))]


def is_probable_prime(n: int, rng: random.Random, rounds: int = 40) -> bool:
    if n < 2 or any(n % p == 0 for p in SMALL_PRIMES):
        return n in SMALL_PRIMES
    d, s = n - 1, 0
    while d % 2 == 0:
        d //= 2
        s += 1
    for _ in range(rounds):
        x = pow(rng.randrange(2, n - 1), d, n)
        if x in (1, n - 1):
            continue
        for _ in range(s - 1):
            x = x * x % n
            if x == n - 1:
                break
        else:
            return False
    return True


def prime_in(lo: int, hi: int, rng: random.Random) -> int:
    """a uniformly drawn probable prime in [lo, hi)"""
    while True:
        c = rng.randrange(lo, hi) | 1
        if c < hi and is_probable_prime(c, rng):
            return c


def paillier_factors(shape: str, rng: random.Random):
    base = shape.replace("_swapped", "")
    if base == "unbalanced":
        p = prime_in(TOP - SLACK, TOP, rng)
        lo = -(-(1 << 2046) // p)
        q = prime_in(lo, lo + SLACK, rng)
    elif base == "small_squares":
        p, q = prime_in(HALF, MID, rng), prime_in(HALF, MID, rng)
    elif base == "min_n":
        p, q = prime_in(HALF, HALF + SLACK, rng), prime_in(HALF, HALF + SLACK, rng)
    elif base == "max_n":
        p, q = prime_in(TOP - SLACK, TOP, rng), prime_in(TOP - SLACK, TOP, rng)
    elif base == "ratio2":
        p, q = prime_in(TOP - SLACK, TOP, rng), prime_in(HALF, HALF + SLACK, rng)
    elif base == "balanced":
        p, q = prime_in(MID, TOP, rng), prime_in(MID, TOP, rng)
    else:
        raise ValueError(shape)
    p, q = max(p, q), min(p, q)
    return (q, p) if shape.endswith("_swapped") else (p, q)


def n_tilde_factors(bits: int, rng: random.Random):
    lo, hi = (HALF, MID) if bits == 2047 else (MID, TOP)
    return prime_in(lo, hi, rng), prime_in(lo, hi, rng)


# per key set: (Paillier shape, N~ bits, small h1) of parties 1..3
KEYSETS = [
    [("unbalanced", 2047, False), ("small_squares_swapped", 2048, False), ("max_n", 2048, True)],
    [("ratio2", 2047, False), ("unbalanced_swapped", 2048, True), ("min_n", 2047, False)],
    [("unbalanced", 2048, False), ("balanced_swapped", 2047, False), ("ratio2_swapped", 2048, True)],
]
SEED = 0xED6E0000


def make_keyset(index: int, rows):
    rng = random.Random(SEED + index)
    a0, a1 = rng.randrange(1, o.Q), rng.randrange(1, o.Q)       # f(x) = a0 + a1 x
    parties = []
    for i, (shape, nt_bits, small_h1) in enumerate(rows, start=1):
        p, q = paillier_factors(shape, rng)
        pt, qt = n_tilde_factors(nt_bits, rng)
        nt, phi = pt * qt, (pt - 1) * (qt - 1)
        h1 = rng.getrandbits(1200) | (1 << 1199) if small_h1 else rng.randrange(2, nt)
        while True:
            xhi = rng.randrange(2, phi)
            if gcd(xhi, phi) == 1:
                break
        parties.append({"i": i, "shape": shape + ("/small_h1" if small_h1 else ""), "p": hex(p), "q": hex(q), "n_tilde": hex(nt),
                        "h1": hex(h1), "h2": hex(pow(h1, xhi, nt)), "x_i": hex((a0 + a1 * i) % o.Q),
                        "p_tilde": hex(pt), "q_tilde": hex(qt), "xhi": hex(xhi)})
    return {"t": 1, "n": len(rows), "secret": hex(a0), "parties": parties}


def main():
    sets = [make_keyset(k, rows) for k, rows in enumerate(KEYSETS)]
    with open(PATH, "w") as f:
        json.dump({"about": "GG20 t=1,n=3 key sets at the edges of the accepted key domain; see make_edge_keys.py", "keysets": sets}, f, indent=1)
        f.write("\n")
    print("wrote", len(sets), "key sets to keys_edge.json")


if __name__ == "__main__":
    main()
