"""Throughput of the GG20 offline stage for any signing set as one device call (tecdsa_gg20_offline_general_batch): elements (one
signer's OfflineStage) per second and executed multiply-accumulates per element for
  (1, 3) with two signers, next to the fused two-signer call (tecdsa_gg20_offline_batch) on the same session count;
  (2, 5) with three signers and (4, 8) with five signers at a few thousand elements per call;
  the Python driver (gg20_general.offline_batch) on a smaller (2, 5) batch, for the before / after.
Per shape: inputs sampled on the device (sample_inputs, TECDSA_DEVICE) and outputs left there, one warm-up call, then `reps` timed
calls (host clock around a call that ends in a stream synchronise), MAC32 from tecdsa_ctx_work, and two sessions of the last call
checked against the size-generic oracle.  The card's name and power limit are read in the same run.  Keys are fresh Shamir sharings
over the fixture Paillier / N~ rows.
    python tools/offline_general_throughput.py [elements] [reps]"""
import json, os, random, subprocess, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
import __graft_entry__ as entry
from oracle import gg20_oracle as o
from tests import test_gg20_offline_general_gpu as tg
from tests.golden import fixtures
pkg = entry.load_package()
from mpecdsa_b200 import DEVICE, gg20, gg20_general


if __name__ == "__main__":      # the oracle check runs in spawned processes, which import this module
    elements = int(sys.argv[1]) if len(sys.argv) > 1 else 3000
    reps = int(sys.argv[2]) if len(sys.argv) > 2 else 2
    card = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    eng = pkg.Engine(0)
    rng = random.Random(0x0FF)
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
        d_sess = torch.tensor(sessions, dtype=torch.int32, device="cuda")
        inp = gg20_general.sample_inputs(eng, ks, T, d_sess, seed=os.urandom(32), mem=DEVICE)
        res, best, mac = timed(lambda: gg20_general.offline_device(eng, ks, T, d_sess, inp, mem=DEVICE))
        h = {f: tg._host(v) for f, v in res.items()}
        picks = [0, ns - 1]
        sub_in = {f: (tg._host(v)[..., [s * T + p for s in picks for p in range(T)], :] if f in gg20_general.STATEMENT_FIELDS or f in gg20_general.PAIR_FIELDS
                      else tg._host(v)[[s * T + p for s in picks for p in range(T)]]) for f, v in inp.items()}
        sub_out = {f: (v[picks] if f == "complete" else v[[s * T + p for s in picks for p in range(T)]]) for f, v in h.items()}
        try:
            tg._check_against_oracle(sub_out, keysets, [sessions[s] for s in picks], sub_in, T, n)
            sample_ok = True
        except AssertionError:
            sample_ok = False
        row = {"t": t, "n": n, "signers": T, "sessions": ns, "elements": ns * T, "seconds_per_call": best, "elements_per_s": ns * T / best,
               "executed_mac32_per_element": mac / (ns * T), "all_complete": bool((h["complete"] == 1).all()), "sample_sessions_match_oracle": sample_ok}
        if T == 2:          # the fused call on the same values, packed into TECDSA_RND_* records
            units, hin = [], {f: tg._host(v) for f, v in inp.items()}
            for u in range(ns * T):
                r = tg._party(hin, u, T, 3)
                units.append(o.UnitRandomness(
                    gamma_i=r.gamma_i, k_i=r.k_i, blind=r.blind, r_k=r.r_k, alice=r.alice, beta_tag_gamma=r.beta_tag_gamma[0], r_gamma=r.r_gamma[0],
                    nonce_gamma_b=r.nonce_gamma_b[0], nonce_gamma_beta=r.nonce_gamma_beta[0], beta_tag_w=r.beta_tag_w[0], r_w=r.r_w[0],
                    nonce_w_b=r.nonce_w_b[0], nonce_w_beta=r.nonce_w_beta[0], l=r.l, ped_s1=r.ped_s1, ped_s2=r.ped_s2, pdl=r.pdl[0],
                    heg_s1=r.heg_s1, heg_s2=r.heg_s2))
            rnd = torch.from_numpy(gg20.pack_randomness(units).view(np.int32)).cuda()
            fs = torch.tensor(sessions, dtype=torch.int32, device="cuda")
            st, R, sg = (torch.zeros(sh, dtype=dt, device="cuda") for sh, dt in (((ns * 2,), torch.uint8), ((ns * 2, 16), torch.int32), ((ns * 2, 8), torch.int32)))
            tv, dg = torch.zeros((ns * 2, 32), dtype=torch.int32, device="cuda"), torch.zeros((ns * 2, 8), dtype=torch.int32, device="cuda")
            _, fbest, fmac = timed(lambda: gg20.offline_raw(eng, ks, fs, ns, rnd, st, R, sg, tv, dg, mem=DEVICE))
            row.update({"fused_seconds_per_call": fbest, "fused_elements_per_s": ns * 2 / fbest, "fused_executed_mac32_per_element": fmac / (ns * 2),
                        "fused_equal": bool((tg._host(R) == h["R"]).all() and (tg._host(sg) == h["sigma"]).all() and (tg._host(st) == h["status"]).all())})
        out["shapes"].append(row)
        print(json.dumps(row), flush=True)
        if (t, n) == (2, 5):        # the Python driver on a smaller batch of the same shape
            small = sessions[:64]
            s_in = gg20_general.sample_inputs(eng, ks, T, small, seed=os.urandom(32))
            args = tg._driver_args(keysets, small, T, n)
            rnd = tg._rnd_of(s_in, T, len(small) * T)
            _, pbest, pmac = timed(lambda: gg20_general.offline_batch(eng, ks, T, *args, rnd))
            _, obest, omac = timed(lambda: gg20_general.offline_device(eng, ks, T, small, s_in))
            drv = {"t": 2, "n": 5, "signers": T, "sessions": len(small), "elements": len(small) * T, "python_driver_elements_per_s": len(small) * T / pbest,
                   "python_driver_mac32_per_element": pmac / (len(small) * T), "one_call_elements_per_s": len(small) * T / obest,
                   "one_call_mac32_per_element": omac / (len(small) * T)}
            out["shapes"].append(drv)
            print(json.dumps(drv), flush=True)
        ks.free()
    print(json.dumps(out))
    eng.close()
