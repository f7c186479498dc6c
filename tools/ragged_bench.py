"""Throughput of independent streams (r8bgpu_batch_process_ragged) next to the same batch driven lock-step.

Each case is one batch of --channels channels with MaxInLen 65536.  The ragged run gives every channel its own block
length per call, drawn from [--min-len, 65536] with a fixed seed; the lock-step runs feed every channel the mean of those
lengths, once with the fused kernels and once with every stage on its own kernel (R8BGPU_NO_FUSION, the chain a ragged
call runs).  Device buffers, asynchronous calls, timed with a device synchronise around --steps calls after --warmup
calls.  Prints one JSON line per case and mode: input samples per second over all channels, ms per call, and kernel
launches per call."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CASES = [(44100.0, 96000.0), (48000.0, 44100.0)]
MAX_IN = 65536


def run(pkg, torch, src, dst, n_ch, lens_seq, ragged, warmup, unfused=False):
    plan = pkg.Plan(src, dst, MAX_IN, 2.0, pkg.ATTEN_24)
    if unfused:
        os.environ["R8BGPU_NO_FUSION"] = "1"
    try:
        b = pkg.Batch(plan, n_ch, 0)
    finally:
        os.environ.pop("R8BGPU_NO_FUSION", None)
    cap = plan.max_out_len
    x = torch.rand((n_ch, MAX_IN), dtype=torch.float64, device="cuda:0") * 2 - 1
    y = torch.empty((n_ch, cap), dtype=torch.float64, device="cuda:0")
    b.set_stream(torch.cuda.current_stream().cuda_stream)
    L = pkg.lib()
    counts = np.empty(n_ch, dtype=np.int32)
    lens_c = [np.ascontiguousarray(v, dtype=np.int32) for v in lens_seq]
    mean_len = int(round(float(np.mean(lens_seq))))

    def call(i):
        if ragged:
            rc = L.r8bgpu_batch_process_ragged(b._h, x.data_ptr(), MAX_IN, lens_c[i].ctypes.data, y.data_ptr(), cap,
                                               cap, counts.ctypes.data)
            if rc < 0:
                raise pkg.R8bGpuError(pkg._err())
            return int(lens_c[i].sum())
        b.process_ptr(x.data_ptr(), MAX_IN, mean_len, y.data_ptr(), cap, cap)
        return mean_len * n_ch

    for i in range(warmup):
        call(i % len(lens_c))
    torch.cuda.synchronize()
    l0 = b.kernel_launches
    t0 = time.perf_counter()
    n_in = 0
    for i in range(warmup, len(lens_c)):
        n_in += call(i)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    steps = len(lens_c) - warmup
    return {"src": src, "dst": dst, "channels": n_ch,
            "mode": "ragged" if ragged else "lockstep, unfused" if unfused else "lockstep",
            "block_len": "%d..%d" % (int(np.min(lens_seq)), int(np.max(lens_seq))) if ragged else mean_len,
            "in_samples_per_s": n_in / dt, "ms_per_call": 1e3 * dt / steps,
            "launches_per_call": (b.kernel_launches - l0) / steps}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--channels", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--min-len", type=int, default=32768)
    ap.add_argument("--seed", type=int, default=1)
    args = ap.parse_args()
    import torch
    from __graft_entry__ import load_package
    pkg = load_package()
    if not torch.cuda.is_available():
        raise SystemExit("ragged_bench: no CUDA device")
    rng = np.random.default_rng(args.seed)
    lens_seq = rng.integers(args.min_len, MAX_IN + 1, size=(args.warmup + args.steps, args.channels))
    gpu = torch.cuda.get_device_name(0)
    for src, dst in CASES:
        for ragged, unfused in ((False, False), (False, True), (True, False)):
            r = run(pkg, torch, src, dst, args.channels, lens_seq, ragged, args.warmup, unfused)
            r["gpu"] = gpu
            print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
