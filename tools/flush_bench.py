"""Cost of ending streams (r8bgpu_batch_flush) and rate of whole-clip resampling (Batch.oneshot_clips).

flush: a batch of --channels channels with MaxInLen 65536 takes one ragged call (lengths drawn from [32768, 65536]),
then every channel is flushed to its default target (device form).  Next to it: the same batch after the same call
takes one ragged call of real zeros, each channel the length of silence its flush feeds (what a caller does without the
flush: upload zero blocks and feed them).  Each is timed with a device synchronise around the call, median of --steps.

clips: --clip-channels clips of 1-10 s at the source rate (seeded lengths), padded to the longest, resampled with
Batch.oneshot_clips from a CUDA tensor (device form) and from a numpy array (host form); rate in input samples per second
(the clips' real lengths), median of --clip-steps runs after one warm-up run.

Prints one JSON line per measurement, with the GPU name and its power limit."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CASES = [(44100.0, 96000.0), (48000.0, 44100.0)]
MAX_IN = 65536


def timed(torch, fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def bench_flush(pkg, torch, src, dst, n_ch, steps, rng):
    plan = pkg.Plan(src, dst, MAX_IN, 2.0, pkg.ATTEN_24)
    b = pkg.Batch(plan, n_ch, 0)
    b.set_stream(torch.cuda.current_stream().cuda_stream)
    L = pkg.lib()
    x = torch.rand((n_ch, MAX_IN), dtype=torch.float64, device="cuda:0") * 2 - 1
    z = torch.zeros((n_ch, MAX_IN), dtype=torch.float64, device="cuda:0")
    cap = max(plan.max_out_len, plan.flush_max_out_len)
    y = torch.empty((n_ch, cap), dtype=torch.float64, device="cuda:0")
    counts = np.empty(n_ch, dtype=np.int32)
    lens = np.ascontiguousarray(rng.integers(32768, MAX_IN + 1, n_ch), dtype=np.int32)
    zl = np.ascontiguousarray([min(MAX_IN, plan.simulate_flush([v])[0]) for v in lens], dtype=np.int32)
    ch = np.arange(n_ch, dtype=np.int32)
    bo = pkg.Buffer.make(y.data_ptr(), pkg.F64, False, cap)

    def feed(lp, src_t):
        if L.r8bgpu_batch_process_ragged(b._h, src_t.data_ptr(), MAX_IN, lp.ctypes.data, y.data_ptr(), cap, cap,
                                         counts.ctypes.data) < 0:
            raise pkg.R8bGpuError(pkg._err())

    def flush():
        if L.r8bgpu_batch_flush(b._h, ch.ctypes.data, n_ch, None, pkg.C.byref(bo), cap, counts.ctypes.data) < 0:
            raise pkg.R8bGpuError(pkg._err())

    t_flush, t_zero, out = [], [], 0
    for i in range(steps + 1):
        b.clear()
        feed(lens, x)
        t = timed(torch, flush)
        out = int(counts.sum())
        b.clear()
        feed(lens, x)
        tz = timed(torch, lambda: feed(zl, z))
        if i > 0:
            t_flush.append(t)
            t_zero.append(tz)
    return {"bench": "flush", "src": src, "dst": dst, "channels": n_ch, "silence_per_channel": int(np.median(zl)),
            "tail_samples": out, "flush_ms": 1e3 * float(np.median(t_flush)),
            "zeros_ragged_call_ms": 1e3 * float(np.median(t_zero))}


def bench_clips(pkg, torch, src, dst, n_ch, steps, rng, host):
    plan = pkg.Plan(src, dst, MAX_IN, 2.0, pkg.ATTEN_24)
    b = pkg.Batch(plan, n_ch, 0)
    lens = rng.integers(int(src), int(10 * src) + 1, n_ch)
    x = np.random.default_rng(0).uniform(-1, 1, (n_ch, int(lens.max())))
    xin = x if host else torch.from_numpy(x).cuda()
    ts = []
    for i in range(steps + 1):
        t = timed(torch, lambda: b.oneshot_clips(xin, lens))
        if i > 0:
            ts.append(t)
    t = float(np.median(ts))
    return {"bench": "oneshot_clips", "form": "host" if host else "device", "src": src, "dst": dst, "clips": n_ch,
            "clip_seconds": "1..10", "in_samples": int(lens.sum()), "ms": 1e3 * t, "in_samples_per_s": lens.sum() / t}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--channels", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--clip-channels", type=int, default=256)
    ap.add_argument("--clip-steps", type=int, default=3)
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--only", choices=["flush", "clips"], default=None)
    args = ap.parse_args()
    import torch
    from __graft_entry__ import load_package
    pkg = load_package()
    if not torch.cuda.is_available():
        raise SystemExit("flush_bench: no CUDA device")
    gpu = torch.cuda.get_device_name(0)
    q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    power = q.stdout.strip() if q.returncode == 0 else "unknown"
    rows = []
    for src, dst in CASES:
        rng = np.random.default_rng(args.seed)
        if args.only in (None, "flush"):
            rows.append(bench_flush(pkg, torch, src, dst, args.channels, args.steps, rng))
        if args.only in (None, "clips"):
            for host in (False, True):
                rows.append(bench_clips(pkg, torch, src, dst, args.clip_channels, args.clip_steps, rng, host))
    for r in rows:
        r["gpu"] = gpu
        r["power_limit"] = power
        print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
