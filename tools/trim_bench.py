"""Cost of drift compensation: a batch whose every channel follows its own rate trim, next to the same trim batch at
f = 1 and to ordinary ragged calls on the nominal plan.

Each case is one batch of --channels channels (default 1024) of 44100->48000 or 48000->44100, CDSPResampler24, MaxInLen
--max-in.  Every mode feeds the same ragged block lengths, drawn per channel and call from [--max-in / 2, --max-in] with a
fixed seed, from device buffers on one stream:
  drift   trim plan (max_trim 2e-4); before every call each channel's factor takes a step of a random walk within
          +-200 ppm (Batch.set_trim), so every channel runs on its own schedule
  trim1   the same trim plan with every factor 1
  ragged  the ordinary plan, r8bgpu_batch_process_ragged
The modes alternate --rounds times; each run times --steps calls after --warmup calls with CUDA events around the calls
and a host clock around the same window ending in a device synchronise (the host clock includes the host-side planning
of every call: set_trim, the per-channel schedules and the record upload).  Prints one JSON line per case and mode with
the median over the rounds and the GPU's name and power limit."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CASES = [(44100.0, 48000.0), (48000.0, 44100.0)]
MAX_TRIM = 2e-4


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0] if r.stdout.strip() else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def walk(rng, f, ppm=200.0, step=20.0):
    """One random-walk step of every channel's factor, kept within +-ppm."""
    return 1.0 + np.clip((f - 1.0) * 1e6 + rng.normal(0.0, step, len(f)), -ppm, ppm) * 1e-6


def run(pkg, torch, plan, mode, n_ch, max_in, lens_seq, warmup, steps):
    """Times ragged calls on a batch of `plan`; mode "drift" walks every channel's factor before each call."""
    b = pkg.Batch(plan, n_ch, 0)
    cap = plan.max_out_len
    x = torch.rand((n_ch, max_in), dtype=torch.float64, device="cuda:0") * 2 - 1
    y = torch.empty((n_ch, cap), dtype=torch.float64, device="cuda:0")
    b.set_stream(torch.cuda.current_stream().cuda_stream)
    L = pkg.lib()
    counts = np.empty(n_ch, dtype=np.int32)
    chans = np.arange(n_ch, dtype=np.int32)
    rng = np.random.default_rng(7)
    f = np.ones(n_ch)
    n_out = [0]

    def call(i):
        if mode == "drift":
            nonlocal f
            f = walk(rng, f)
            b.set_trim(chans, f)
        lens = lens_seq[i % len(lens_seq)]
        if L.r8bgpu_batch_process_ragged(b._h, x.data_ptr(), max_in, lens.ctypes.data, y.data_ptr(), cap, cap,
                                         counts.ctypes.data) != 0:
            raise pkg.R8bGpuError(pkg._err())
        n_out[0] += int(counts.sum())

    for i in range(warmup):
        call(i)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    n_out[0] = 0
    t0 = time.perf_counter()
    e0.record()
    for i in range(steps):
        call(warmup + i)
    e1.record()
    torch.cuda.synchronize()
    wall = (time.perf_counter() - t0) / steps * 1e3
    ev = e0.elapsed_time(e1) / steps
    n_in = sum(int(lens_seq[(warmup + i) % len(lens_seq)].sum()) for i in range(steps))
    return dict(ms_per_call_events=ev, ms_per_call_wall=wall, in_samples_per_s=n_in / (wall * 1e-3 * steps),
                out_per_call=n_out[0] / steps, groups=b.channel_groups)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--channels", type=int, default=1024)
    ap.add_argument("--max-in", type=int, default=16384)
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=6)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    import torch
    import __graft_entry__
    pkg = __graft_entry__.load_package()
    if not torch.cuda.is_available() or pkg.device_count() < 1:
        raise SystemExit("trim_bench: no CUDA device")
    gpu = gpu_info()
    rng = np.random.default_rng(1)
    lens_seq = [np.ascontiguousarray(rng.integers(a.max_in // 2, a.max_in + 1, a.channels), dtype=np.int32)
                for _ in range(a.warmup + a.steps)]
    for src, dst in CASES:
        res = {m: [] for m in ("drift", "trim1", "ragged")}
        for _ in range(a.rounds):
            for m in res:
                plan = pkg.Plan(src, dst, a.max_in, 2.0, pkg.ATTEN_24) if m == "ragged" else \
                    pkg.Plan.trim(src, dst, a.max_in, 2.0, pkg.ATTEN_24, MAX_TRIM)
                res[m].append(run(pkg, torch, plan, m, a.channels, a.max_in, lens_seq, a.warmup, a.steps))
        for m, rs in res.items():
            med = {k: float(np.median([r[k] for r in rs])) for k in rs[0]}
            med["ms_per_call_wall_all"] = [round(r["ms_per_call_wall"], 4) for r in rs]
            print(json.dumps(dict(case="%g->%g" % (src, dst), mode=m, channels=a.channels, max_in=a.max_in, gpu=gpu,
                                  **med)), flush=True)


if __name__ == "__main__":
    main()
