"""Throughput of GG18 signing as one device call (tecdsa_gg18_signing_batch): sessions and elements (one signer's signing) per second
and executed multiply-accumulates per element for (1, 3) with two signers, (2, 5) with three and (4, 8) with five at about `elements`
elements per call, and gg18.sign_batch (the Python driver of about 25 batch calls) on a 64-session (2, 5) batch next to the one call
on the same inputs.  Per shape: inputs sampled on the device (sample_inputs, TECDSA_DEVICE) and outputs left there, one warm-up call,
then the best of `reps` timed calls (host clock around a call that ends in a stream synchronise), MAC32 from tecdsa_ctx_work, and two
sessions of the last call checked against the party-by-party restatement (tests/gg18_signing_oracle.py).  The card's name and power
limit are read in the same run.  Keys are fresh Shamir sharings over the fixture Paillier rows.
    python tools/gg18_signing_throughput.py [elements] [reps]"""
import json, os, random, subprocess, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
import __graft_entry__ as entry
from tests import test_gg18_signing_gpu as tg
from tests.golden import fixtures
pkg = entry.load_package()
from mpecdsa_b200 import DEVICE, gg18, gg20


if __name__ == "__main__":      # the oracle check runs in spawned processes, which import this module
    elements = int(sys.argv[1]) if len(sys.argv) > 1 else 2000
    reps = int(sys.argv[2]) if len(sys.argv) > 2 else 2
    card = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    eng = pkg.Engine(0)
    rng = random.Random(0x18)
    fix = tg._rows()
    out = {"card_and_power_limit": card, "timed_calls": reps, "shapes": []}

    def timed(fn):
        fn()                                                      # warm-up
        times, work = [], []
        for _ in range(reps):
            eng.work(reset=True)
            t0 = time.perf_counter()
            res = fn()
            eng.sync()
            times.append(time.perf_counter() - t0)
            work.append(eng.work())
        return res, min(times), work[-1]

    for t, n, T in ((1, 3, 2), (2, 5, 3), (4, 8, 5)):
        keysets = fixtures.load_all_keysets() if n == 3 else [tg._key(fix[k * n:(k + 1) * n], t, n, rng) for k in range(len(fix) // n)]
        ks = gg20.KeySets(eng, keysets)
        ns = elements // T
        sessions = [[s % len(keysets)] + rng.sample(range(n), T) for s in range(ns)]
        msg = tg._messages(ns, t * 100 + n)
        d_sess = torch.tensor(sessions, dtype=torch.int32, device="cuda")
        d_msg = torch.from_numpy(pkg.ints_to_limbs(msg, 8).view(np.int32)).cuda()
        inp = gg18.sample_inputs(eng, ks, T, d_sess, seed=os.urandom(32), mem=DEVICE)
        res, best, mac = timed(lambda: gg18.sign_device(eng, ks, T, d_sess, d_msg, inp, mem=DEVICE))
        h = {f: tg._host(v) for f, v in res.items()}
        picks = [0, ns - 1]
        try:
            tg._check_against_oracle(tg._slice_out(h, picks, T), keysets, [sessions[s] for s in picks], tg._slice({f: tg._host(v) for f, v in inp.items()}, picks, T),
                                     [msg[s] for s in picks], T)
            sample_ok = True
        except AssertionError:
            sample_ok = False
        row = {"t": t, "n": n, "signers": T, "sessions": ns, "elements": ns * T, "seconds_per_call": best, "sessions_per_s": ns / best,
               "elements_per_s": ns * T / best, "executed_mac32_per_element": mac / (ns * T), "all_complete": bool((h["complete"] == 1).all()),
               "sample_sessions_match_oracle": sample_ok}
        out["shapes"].append(row)
        print(json.dumps(row), flush=True)
        if (t, n) == (2, 5):        # the Python driver on a smaller batch of the same shape, and the one call on the same inputs
            small, smsg = sessions[:64], msg[:64]
            s_in = gg18.sample_inputs(eng, ks, T, small, seed=os.urandom(32))
            args = tg._sign_batch_args(keysets, small, T, n, s_in, smsg)
            _, pbest, pmac = timed(lambda: gg18.sign_batch(eng, ks, T, *args))
            _, obest, omac = timed(lambda: gg18.sign_device(eng, ks, T, small, smsg, s_in))
            drv = {"t": 2, "n": 5, "signers": T, "sessions": len(small), "elements": len(small) * T, "python_driver_elements_per_s": len(small) * T / pbest,
                   "python_driver_mac32_per_element": pmac / (len(small) * T), "one_call_elements_per_s": len(small) * T / obest,
                   "one_call_mac32_per_element": omac / (len(small) * T)}
            out["shapes"].append(drv)
            print(json.dumps(drv), flush=True)
        ks.free()
    print(json.dumps(out))
    eng.close()
