"""Crops of long clips: a training-style workload of 64 clips of 10 min at 48000 Hz -> 16000 Hz (float32 CUDA tensors,
MaxInLen 65536, CDSPResampler24, 1024 lanes) with one random 4 s output crop per clip.

  (a) crops          Batch.oneshot_crops
  (b) long+slice     Batch.oneshot_long of the whole clips, then each crop sliced out
  (c) grad crops     resample_crops forward and backward
      grad clips     resample_clips forward and backward on the loss of the sliced crops

Times are CUDA events around each arm (every call finishes before it returns).  One warm-up per arm, then the arms
alternate over --reps repetitions; the best and the median are printed.  The outputs of (a) and (b) and the gradients
of the two (c) arms must be identical (the gradients as numbers), or the run stops.  The GPU's name, power limit and max
SM clock are read in the same run.  One JSON line per arm."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from __graft_entry__ import load_package  # noqa: E402


def gpu_line():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # the numbers still stand; say what is missing
        return "unknown (%s)" % e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clips", type=int, default=64)
    ap.add_argument("--minutes", type=float, default=10.0)
    ap.add_argument("--crop-seconds", type=float, default=4.0)
    ap.add_argument("--lanes", type=int, default=1024)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    import torch
    pkg = load_package()
    gpu = gpu_line()
    src, dst = 48000.0, 16000.0
    plan = pkg.Plan(src, dst, 65536, 2.0, pkg.ATTEN_24)
    b = pkg.Batch(plan, a.lanes, device=0)
    n = int(src * a.minutes * 60)
    g0 = torch.Generator(device="cuda").manual_seed(1)
    x = torch.rand((a.clips, n), dtype=torch.float32, device="cuda", generator=g0) * 2 - 1
    lens = np.full(a.clips, n, dtype=np.int64)
    op = plan.default_target(n)
    w = int(dst * a.crop_seconds)
    rng = np.random.default_rng(2)
    o0 = rng.integers(0, op - w + 1, a.clips)
    crops = np.stack([np.arange(a.clips), o0, o0 + w], axis=1).astype(np.int64)
    gy = torch.rand((a.clips, w), dtype=torch.float32, device="cuda", generator=g0) * 2 - 1

    out = {}

    def arm_crops():
        out["a"] = b.oneshot_crops(x, crops, lens)

    def arm_long():
        y, _ = b.oneshot_long(x, lens)
        out["b"] = torch.stack([y[r, s:e] for r, s, e in crops])

    def arm_grad_crops():
        xg = x.detach().requires_grad_(True)
        (pkg.resample_crops(b, xg, crops, lens) * gy).sum().backward()
        out["c"] = xg.grad

    def arm_grad_clips():
        xg = x.detach().requires_grad_(True)
        y = pkg.resample_clips(b, xg, lens)
        sl = torch.stack([y[r, s:e] for r, s, e in crops])
        (sl * gy).sum().backward()
        out["d"] = xg.grad

    arms = [("crops", arm_crops), ("long+slice", arm_long), ("grad crops", arm_grad_crops), ("grad clips", arm_grad_clips)]
    times = {k: [] for k, _ in arms}
    for k, f in arms:  # warm-up
        f()
    if not torch.equal(out["a"], out["b"]):
        sys.exit("crops differ from the sliced whole-clip output")
    if not torch.equal(out["c"], out["d"]):  # == on numbers: -0 equals +0
        sys.exit("crop gradients differ from the whole-clip gradients")
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(a.reps):
        for k, f in arms:
            torch.cuda.synchronize()
            ev0.record()
            f()
            ev1.record()
            torch.cuda.synchronize()
            times[k].append(ev0.elapsed_time(ev1))
    for k, _ in arms:
        t = sorted(times[k])
        print(json.dumps({"arm": k, "best_ms": round(t[0], 2), "median_ms": round(t[len(t) // 2], 2),
                          "clips": a.clips, "clip_samples": n, "crop_outputs": w, "lanes": a.lanes, "gpu": gpu}))


if __name__ == "__main__":
    main()
