"""Cost of the seeded sampler at the benchmark's size (8 192 sessions = 16 384 units over the 8 fixture key sets), one JSON line:
  (a) kernel time of tecdsa_gg20_sample_randomness beside the offline stage's kernels, from the per-launch profile of one step;
  (b) end-to-end phases/s of "host rnd -> H2D -> offline -> records -> D2H" (tecdsa_gg20_offline_records on pinned buffers)
      against "seed -> sample on the device -> offline -> records -> D2H", alternated, with the spread of each;
the card's name and power limit are read in the same run.
    python tools/prof_sampler.py [--sessions 8192] [--steps 5] [--warmup 1]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import __graft_entry__ as entry
from tests.golden import fixtures


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sessions", type=int, default=8192)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()
    pkg = entry.load_package()
    from mpecdsa_b200 import gg20
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True).stdout.strip()
    eng = pkg.Engine(0)
    keysets = fixtures.load_all_keysets()
    ks = gg20.KeySets(eng, keysets)
    n, U = a.sessions, 2 * a.sessions
    sessions, rnd = gg20.synthetic_batch(keysets, n, 0xB2000005)
    pin = lambda arr: torch.from_numpy(arr).pin_memory().numpy()
    h_sess, h_rnd = pin(sessions), pin(rnd)
    h_rec = torch.zeros((1, U, pkg.REC_BYTES), dtype=torch.uint8).pin_memory()
    Z = lambda *shape, dt=torch.int32: torch.zeros(shape, dtype=dt, device="cuda")
    d_sess = torch.from_numpy(sessions.view(np.int32)).cuda()
    d_rnd, d_sst, d_st, d_R, d_sig, d_t, d_dig = Z(U, gg20.RND_LIMBS), Z(U, dt=torch.uint8), Z(U, dt=torch.uint8), Z(U, 16), Z(U, 8), Z(U, 32), Z(U, 8)
    d_rec = Z(U, pkg.REC_BYTES, dt=torch.uint8)
    seeds = iter(range(1, 1 << 30))

    def host_rnd():
        eng.offline_records(ks, None, h_sess, n, h_rnd, h_rec.numpy(), pkg.HOST)
        return h_rec[0, :, 0]

    def seeded():
        gg20.sample_randomness(eng, ks, d_sess, seed=next(seeds).to_bytes(32, "little"), mem=pkg.DEVICE, rnd=d_rnd, status=d_sst)
        gg20.offline_raw(eng, ks, d_sess, n, d_rnd, d_st, d_R, d_sig, d_t, d_dig, mem=pkg.DEVICE)
        eng.pack_records(d_st, d_R, d_sig, d_t, d_dig, d_rnd, U, d_rec)
        h_rec[0].copy_(d_rec, non_blocking=True)
        eng.sync()
        return h_rec[0, :, 0]

    def timed(fn):
        t0 = time.perf_counter()
        st = fn()
        dt = time.perf_counter() - t0
        assert not st.numpy().any(), "a unit failed"
        return dt

    for _ in range(a.warmup):
        timed(host_rnd); timed(seeded)
    assert not d_sst.cpu().numpy().any()
    t = {"host_rnd": [], "seeded": []}
    for _ in range(a.steps):
        t["host_rnd"].append(timed(host_rnd)); t["seeded"].append(timed(seeded))
    prof = eng.profile_step(seeded)
    sample_ms = prof.get("gg20_sample", {"ms": float("nan")})["ms"]
    total_ms = sum(v["ms"] for v in prof.values())
    out = {"card": card, "sessions": n, "units": U, "key_sets": len(keysets), "steps": a.steps, "warmup": a.warmup,
           "kernel_ms": {"gg20_sample": sample_ms, "all_kernels_of_the_step": total_ms, "share": sample_ms / total_ms},
           "e2e": {k: {"phases_per_s_median": U / statistics.median(v), "phases_per_s_min": U / max(v), "phases_per_s_max": U / min(v),
                       "seconds": [round(x, 4) for x in v]} for k, v in t.items()}}
    print(json.dumps(out))
    ks.free()
    eng.close()


if __name__ == "__main__":
    main()
