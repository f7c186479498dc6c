"""Gradients through long clips: Batch.oneshot_adjoint against Batch.oneshot_long on the same clips, on a 1024-lane batch,
device form, float64 CUDA tensors:

  48000-44100    8 clips of 30 s, 48000 -> 44100 (BlockConv 2x, whole-stepping interpolator)
  44100-96000    8 clips of 30 s, 44100 -> 96000 (the flagship chain)
  48000-47999    8 clips of 30 s, 48000 -> 47999 (order-2 interpolator)
  96000-48000    8 clips of 30 s, 96000 -> 48000 (block-exact 1/2)
  192000-44100   8 clips of 30 s, 192000 -> 44100 (half-band decimators)

Times are CUDA events around each call (both finish before they return); the arms alternate over --reps repetitions and the
best of each is printed with its input samples per second, the dot-product ratio |<Ax, g> - <x, A^T g>| / (|Ax| |g|) and the
GPU's name, power limit and max SM clock.  One JSON line per workload."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from __graft_entry__ import load_package  # noqa: E402

WORKLOADS = [("48000-44100", 48000.0, 44100.0), ("44100-96000", 44100.0, 96000.0), ("48000-47999", 48000.0, 47999.0),
             ("96000-48000", 96000.0, 48000.0), ("192000-44100", 192000.0, 44100.0)]


def gpu_line():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # the numbers still stand; say what is missing
        return "unknown (%s)" % e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=30.0)
    ap.add_argument("--clips", type=int, default=8)
    ap.add_argument("--lanes", type=int, default=1024)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    import torch
    pkg = load_package()
    gpu = gpu_line()
    for name, src, dst in WORKLOADS:
        plan = pkg.Plan(src, dst, 65536, 2.0, pkg.ATTEN_24)
        b = pkg.Batch(plan, a.lanes, device=0)
        n = int(src * a.seconds)
        g0 = torch.Generator(device="cuda").manual_seed(1)
        x = torch.rand((a.clips, n), dtype=torch.float64, device="cuda", generator=g0) * 2 - 1
        lens = np.full(a.clips, n, dtype=np.int64)
        y, oplens = b.oneshot_long(x, lens)
        g = torch.rand(y.shape, dtype=torch.float64, device="cuda", generator=g0) * 2 - 1
        gx = b.oneshot_adjoint(g, lens, oplens, width=n)
        lhs = (y * g).sum(dim=1)
        rhs = (x * gx).sum(dim=1)
        ratio = float(((lhs - rhs).abs() / (y.norm(dim=1) * g.norm(dim=1))).max())
        best = {"forward": float("inf"), "adjoint": float("inf")}
        for _ in range(a.reps):
            for arm in ("forward", "adjoint"):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                if arm == "forward":
                    b.oneshot_long(x, lens)
                else:
                    b.oneshot_adjoint(g, lens, oplens, width=n)
                e1.record()
                e1.synchronize()
                best[arm] = min(best[arm], e0.elapsed_time(e1))
        samples = float(a.clips * n)
        print(json.dumps({"workload": name, "clips": a.clips, "seconds": a.seconds, "lanes": a.lanes,
                          "forward_ms": round(best["forward"], 2), "adjoint_ms": round(best["adjoint"], 2),
                          "adjoint_over_forward": round(best["adjoint"] / best["forward"], 2),
                          "adjoint_msamples_per_s": round(samples / best["adjoint"] / 1e3, 1),
                          "dot_ratio": ratio, "gpu": gpu}), flush=True)


if __name__ == "__main__":
    main()
