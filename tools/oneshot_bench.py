"""Long clips on the whole GPU: Batch.oneshot_long on a 1024-lane batch (device and host forms) against the one-channel-
per-clip path (Batch.oneshot_clips on a batch of n_clips channels), on three file-converter workloads:

  stereo   one stereo 10-minute 44100 -> 96000 clip, float32 in and out
  dsd      one 2-channel DSD64 clip (2 minutes) -> 88200 float32
  s16      64 clips of 1-10 minutes at 48000 -> 44100, int16 with flat TPDF dither

Times are a host clock around the synchronising call; the arms alternate over --reps repetitions and the best of each is
printed, with the outputs of every arm checked bit for bit against each other.  One JSON line per workload and arm."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from __graft_entry__ import load_package  # noqa: E402


def gpu_line():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # the numbers still stand; say what is missing
        return "unknown (%s)" % e


def workloads(rng, minutes_scale):
    pkg = load_package()
    s = minutes_scale
    n = int(44100 * 600 * s)
    yield "stereo", (44100.0, 96000.0, 65536), rng.uniform(-0.9, 0.9, (2, n)).astype(np.float32), \
        dict(fmt=pkg.F32, out_fmt=pkg.F32), None
    n = int(2822400 * 120 * s) // 8 * 8
    yield "dsd", (2822400.0, 88200.0, 65536), rng.integers(0, 256, (2, n // 8), dtype=np.uint8), \
        dict(fmt=pkg.DSD_LSB, out_fmt=pkg.F32, in_scale=0.5), None
    lens = (rng.integers(60, 601, 64) * 48000 * s).astype(np.int64)
    x = np.zeros((64, int(lens.max())), dtype=np.int16)
    for r, v in enumerate(lens):
        x[r, :v] = rng.integers(-20000, 20000, int(v), dtype=np.int16)
    yield "s16", (48000.0, 44100.0, 65536), (x, lens), dict(fmt=pkg.S16, out_fmt=pkg.S16), [1000 + r for r in range(64)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lanes", type=int, default=1024)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--scale", type=float, default=1.0, help="clip lengths relative to the workloads above")
    a = ap.parse_args()
    import torch
    pkg = load_package()
    print(json.dumps({"gpu": gpu_line(), "lanes": a.lanes}), flush=True)
    rng = np.random.default_rng(1)
    for name, (src, dst, mil), data, kw, seeds in workloads(rng, a.scale):
        x, lens = data if isinstance(data, tuple) else (data, None)
        plan = pkg.Plan(src, dst, mil, 2.0, pkg.ATTEN_24)
        n_clips = x.shape[0]
        spe = 8 if kw["fmt"] in (pkg.DSD_LSB, pkg.DSD_MSB) else 1
        if lens is None:
            lens = np.full(n_clips, x.shape[1] * spe, dtype=np.int64)
        xd = torch.from_numpy(x).cuda()
        lanes = pkg.Batch(plan, a.lanes, device=0)
        twin = pkg.Batch(plan, n_clips, device=0)
        dith = None if seeds is None else [pkg.Dither.make(s) for s in seeds]

        def twin_run(xx):
            if dith is not None:
                twin.set_dither(list(range(n_clips)), seeds)
            y, _ = twin.oneshot_clips(xx, lens, **kw)
            return y

        arms = {
            "oneshot_long_device": lambda: lanes.oneshot_long(xd, lens, dither=dith, **kw)[0],
            "oneshot_long_host": lambda: lanes.oneshot_long(x, lens, dither=dith, **kw)[0],
            "oneshot_clips_device": lambda: twin_run(xd),
            "oneshot_clips_host": lambda: twin_run(x),
        }
        best = {k: float("inf") for k in arms}
        outs = {}
        for rep in range(a.reps + 1):  # the first pass warms every shape up
            for k, fn in arms.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                y = fn()
                torch.cuda.synchronize()
                dt = time.perf_counter() - t0
                if rep > 0:
                    best[k] = min(best[k], dt)
                y = y.cpu().numpy() if hasattr(y, "cpu") else y
                outs[k] = y[:, :int(y.shape[1])]
        ref = outs["oneshot_clips_host"]
        same = all(o.shape == ref.shape and o.tobytes() == ref.tobytes() for o in outs.values())
        segs, n_calls = plan.simulate_oneshot(a.lanes, lens)
        for k in arms:
            print(json.dumps({"workload": name, "arm": k, "seconds": round(best[k], 4),
                              "input_samples_per_s": float(lens.sum()) / best[k], "bit_identical": same,
                              "segments": len(segs), "ragged_calls": n_calls if k.startswith("oneshot_long") else None}),
                  flush=True)
        del lanes, twin, xd


if __name__ == "__main__":
    main()
