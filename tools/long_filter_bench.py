#!/usr/bin/env python3
"""Device-resident rate of a long-filter chain on the large-tile BlockConvolver (DESIGN.md K1c), verified like bench.py.

Default: 1024 channels, 48000 -> 16000, CDSPResampler24 at a 0.5 % transition band (one 1/3 BlockConvolver with 8507
taps on 65536-point tiles), 65536-frame blocks.  K steps are timed with CUDA events on the launch stream; afterwards every
call the batch has seen is replayed through the oracle on four sampled channels (bench.verify_against_oracle: counts
equal, <= 32 eps max, <= 4 eps rms).  --profile adds a separate torch.profiler pass with the device time of every kernel
per step.  Prints one JSON line; writes nothing.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--src", type=float, default=48000.0)
    ap.add_argument("--dst", type=float, default=16000.0)
    ap.add_argument("--tb", type=float, default=0.5)
    ap.add_argument("--atten", type=float, default=180.15)
    ap.add_argument("--extfft", type=int, default=0)
    ap.add_argument("--channels", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=4)
    ap.add_argument("--profile", action="store_true")
    a = ap.parse_args()

    import numpy as np
    import torch
    import bench
    from __graft_entry__ import load_package
    pkg = load_package()
    if not torch.cuda.is_available() or pkg.device_count() < 1:
        raise SystemExit("long_filter_bench.py: no CUDA device -- the engine has no CPU fallback")
    block, n_ch = bench.BLOCK, a.channels
    t0 = time.perf_counter()
    plan = pkg.Plan(a.src, a.dst, block, a.tb, a.atten, extfft=a.extfft)
    batch = pkg.Batch(plan, n_ch, 0)
    create_s = time.perf_counter() - t0
    cap = (plan.max_out_len + 7) // 8 * 8
    xs = [torch.from_numpy(bench.synth_block(n_ch, block, 1000 + i)).cuda() for i in range(2)]
    out = torch.empty((n_ch, cap), dtype=torch.float64, device="cuda")
    stream = torch.cuda.current_stream()
    batch.set_stream(stream.cuda_stream)
    calls = []

    def step(i):
        calls.append(i & 1)
        return batch.process_ptr(xs[i & 1].data_ptr(), block, block, out.data_ptr(), cap, cap)

    for i in range(max(3, a.warmup)):
        step(i)
    torch.cuda.synchronize()
    sampler = bench.ClockSampler(0)
    sampler.start()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    counts = [step(i) for i in range(a.steps)]
    e1.record(stream)
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1)
    clocks = sampler.stop()
    check_ch = sorted(set([0, n_ch // 3, (2 * n_ch) // 3, n_ch - 1]))
    got_last = out[check_ch, :counts[-1]].cpu().numpy()
    check_x = [x[check_ch].cpu().numpy() for x in xs]
    verified = bench.verify_against_oracle(a.src, a.dst, a.tb, a.atten, a.extfft, check_x, list(calls), got_last, check_ch)

    kernels = None
    if a.profile:
        k = max(1, min(a.steps, 10))
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for i in range(k):
                step(i)
            torch.cuda.synchronize()
        kernels = {}
        for e in prof.key_averages():
            if getattr(e, "self_device_time_total", 0) > 0:
                kernels[e.key[:90]] = {"ms_per_step": e.self_device_time_total / 1e3 / k, "launches_per_step": e.count / k}

    gpu = None
    try:  # the board and its power limit are part of the number
        import subprocess
        gpu = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=10).stdout.strip()
    except Exception:
        pass
    print(json.dumps({
        "metric": "input Msamples/s, fp64 %g->%g, TransBand %g %%, %g dB, extfft %d" % (a.src, a.dst, a.tb, a.atten, a.extfft),
        "value": 1e-6 * n_ch * block * a.steps / (ms * 1e-3), "unit": "Msamples/s", "ms_per_step": ms / a.steps,
        "channels": n_ch, "block_frames": block, "steps": a.steps, "stage_kernels": batch.stage_kernels(),
        "device_state_bytes": batch.device_bytes, "batch_create_s": create_s, "gpu": gpu, "clocks": clocks,
        "verified": bool(verified["ok"]), "verification": verified, "kernels": kernels}))
    return 0


if __name__ == "__main__":
    sys.exit(main())
