"""Writes n_tilde_64.json: 64 distinct N~ prime pairs (1024-bit primes, 2048-bit products) for key generation at n = 64, made by
tests/keygen_group.py::prime_pair from the seeds 0x6400..0x643f.  Run from the repository root: python -m tests.golden.make_n_tilde_64"""
import json
import os
from concurrent.futures import ProcessPoolExecutor

from tests import keygen_group as kgg

SEEDS = [0x6400 + i for i in range(64)]


def main():
    with ProcessPoolExecutor() as pool:
        pairs = list(pool.map(kgg.prime_pair, SEEDS))
    doc = {"seeds": SEEDS, "pairs": [[format(p, "x"), format(q, "x")] for p, q in pairs]}
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "n_tilde_64.json"), "w") as f:
        json.dump(doc, f, indent=0)
        f.write("\n")


if __name__ == "__main__":
    main()
