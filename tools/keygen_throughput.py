"""Throughput of GG20 key generation as one device call (tecdsa_gg20_keygen_batch): parties per second for (t, n) = (1, 3) and (2, 5) at
`groups` groups per call (default 2048), inputs sampled on the device (keygen.sample_randomness, TECDSA_DEVICE) and every output left on
the device.  Per shape: one warm-up call, then `reps` timed calls (host clock around a call that ends in a stream synchronise), the
multiply-accumulates the big-integer kernels executed (tecdsa_ctx_work) per party, and a check of a 64-element sample of the last call
against the party-by-party group oracle (tests/keygen_group.py).  The card's name and power limit are read in the same run.
Paillier and N~ primes cycle through the 24 fixture key rows: prime generation is not part of the call, and the work of a party does
not depend on which primes it holds.
    python tools/keygen_throughput.py [groups] [reps]"""
import json, os, subprocess, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import __graft_entry__ as entry
from tests import keygen_group as kgg
from tests.golden import fixtures
pkg = entry.load_package()
from mpecdsa_b200 import keygen

groups = int(sys.argv[1]) if len(sys.argv) > 1 else 2048
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 3
SAMPLE = 64
card = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
eng = pkg.Engine(0)
rows = [lk for ks in fixtures.load_all_keysets() for lk in ks]
out = {"card_and_power_limit": card, "groups_per_call": groups, "timed_calls": reps, "shapes": []}
for t, n in ((1, 3), (2, 5)):
    E = groups * n
    paillier = [(rows[e % 12].dk.p, rows[e % 12].dk.q) for e in range(E)]
    n_tilde = [(rows[12 + e % 12].dk.p, rows[12 + e % 12].dk.q) for e in range(E)]
    rec = keygen.sample_randomness(eng, t, n, n_tilde, os.urandom(32), mem=pkg.DEVICE)
    res = keygen.keygen_batch(eng, t, n, paillier, n_tilde, rec, mem=pkg.DEVICE)            # warm-up
    times, work = [], []
    for _ in range(reps):
        eng.work(reset=True)
        t0 = time.perf_counter()
        res = keygen.keygen_batch(eng, t, n, paillier, n_tilde, rec, mem=pkg.DEVICE)
        times.append(time.perf_counter() - t0)
        work.append(eng.work())
    ok = bool((res.status == 0).all() and (res.complete == 1).all())
    # 64-element sample: evenly spaced whole groups, every output compared with the group oracle
    picks = np.linspace(0, groups - 1, (SAMPLE + n - 1) // n).round().astype(int)
    host = {f: keygen._host(v) for f, v in res.out.items()}
    I = lambda a: int.from_bytes(np.ascontiguousarray(a).tobytes(), "little")
    sample_ok = True
    for g in picks:
        es = range(g * n, g * n + n)
        r = {f: keygen._host(v[g * n:g * n + n]) for f, v in rec.items()}
        rnd = [{"u": I(r["u"][i]), "coeffs": [I(c) for c in r["coeffs"][i]], "blind": I(r["blind"][i]), "h1": I(r["h1"][i]), "xhi": I(r["xhi"][i]),
                "cdl_nonce": tuple(I(c) for c in r["cdl_nonce"][i]), "dlog_nonce": I(r["dlog_nonce"][i])} for i in range(n)]
        keys, status, bad = kgg.keygen_group(t, n, [(paillier[e], n_tilde[e]) for e in es], rnd)
        got_y = host["y"][g]
        sample_ok &= list(res.status[list(es)]) == status and list(res.bad_actors[list(es)]) == bad
        sample_ok &= (I(got_y[:8]), I(got_y[8:])) == keys[0].y_sum_s
        for i, e in enumerate(es):
            lk = keys[i]
            sample_ok &= I(host["x_i"][e]) == lk.x_i and I(host["n"][e]) == lk.paillier_key_vec[i].n
            sample_ok &= [(I(p[:8]), I(p[8:])) for p in host["vss"][e]] == lk.vss_commitments
            sample_ok &= [I(v) for v in host["dlog_st"][e]] == [lk.h1_h2_n_tilde_vec[i].N, lk.h1_h2_n_tilde_vec[i].g, lk.h1_h2_n_tilde_vec[i].ni]
            sample_ok &= (I(host["pk"][g, i, :8]), I(host["pk"][g, i, 8:])) == lk.pk_vec[i]
    best = min(times)
    out["shapes"].append({"t": t, "n": n, "parties": E, "seconds_per_call": times, "parties_per_s": E / best, "groups_per_s": groups / best,
                          "executed_mac32_per_party": work[-1] / E, "executed_tmac32_per_s": work[-1] / best / 1e12,
                          "all_complete": ok, "sample_elements_checked": int(len(picks) * n), "sample_matches_oracle": bool(sample_ok)})
    print(json.dumps(out["shapes"][-1]), flush=True)
print(json.dumps(out))
eng.close()
