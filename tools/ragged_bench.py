"""Throughput of independent streams (r8bgpu_batch_process_ragged) next to the same batch driven lock-step.

Each case is one batch of --channels channels with MaxInLen 65536.  The ragged run gives every channel its own block
length per call, drawn from [--min-len, 65536] with a fixed seed; the lock-step runs feed every channel the mean of those
lengths, once with the fused kernels and once with every stage on its own kernel (R8BGPU_NO_FUSION, the chain a ragged
call runs).  Device buffers, asynchronous calls, timed with a device synchronise around --steps calls after --warmup
calls.  Prints one JSON line per case and mode: input samples per second over all channels, ms per call, and kernel
launches per call.

--format f32 / s16 runs only the ragged mode, with typed buffers of that format in and out
(r8bgpu_batch_process_ragged_fmt; f64 keeps the plain fp64 entry points).  --host runs only the ragged mode through the
host form (r8bgpu_batch_process_host_ragged / _host_ragged_fmt) on pinned host buffers, so the copies over PCIe are
inside the timed region; the line then also gives the PCIe bytes moved per input sample."""
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

CASES = [(44100.0, 96000.0), (48000.0, 44100.0)]
MAX_IN = 65536
FORMATS = {"f64": ("float64", 0), "f32": ("float32", 1), "s16": ("int16", 2)}  # numpy dtype, r8bgpu_sample_format


def run(pkg, torch, src, dst, n_ch, lens_seq, ragged, warmup, unfused=False, fmt="f64", host=False):
    plan = pkg.Plan(src, dst, MAX_IN, 2.0, pkg.ATTEN_24)
    if unfused:
        os.environ["R8BGPU_NO_FUSION"] = "1"
    try:
        b = pkg.Batch(plan, n_ch, 0)
    finally:
        os.environ.pop("R8BGPU_NO_FUSION", None)
    cap = plan.max_out_len
    dtype, code = FORMATS[fmt]
    esize = np.dtype(dtype).itemsize
    amp = 20000.0 if fmt == "s16" else 1.0
    if host:
        x, y = b.host_alloc(MAX_IN, dtype), b.host_alloc(cap, dtype)
        x[:] = ((np.random.default_rng(0).random((n_ch, MAX_IN)) * 2 - 1) * amp).astype(dtype)
        x_ptr, y_ptr = x.ctypes.data, y.ctypes.data
    else:
        x = ((torch.rand((n_ch, MAX_IN), dtype=torch.float64, device="cuda:0") * 2 - 1) * amp).to(getattr(torch, dtype))
        y = torch.empty((n_ch, cap), dtype=getattr(torch, dtype), device="cuda:0")
        x_ptr, y_ptr = x.data_ptr(), y.data_ptr()
    b.set_stream(torch.cuda.current_stream().cuda_stream)
    L = pkg.lib()
    counts = np.empty(n_ch, dtype=np.int32)
    lens_c = [np.ascontiguousarray(v, dtype=np.int32) for v in lens_seq]
    mean_len = int(round(float(np.mean(lens_seq))))
    bi, bo = pkg.Buffer.make(x_ptr, code, False, MAX_IN), pkg.Buffer.make(y_ptr, code, False, cap)
    n_out = [0]

    def call(i):
        if ragged:
            lp, cp = lens_c[i].ctypes.data, counts.ctypes.data
            if fmt == "f64":
                fn = L.r8bgpu_batch_process_host_ragged if host else L.r8bgpu_batch_process_ragged
                rc = fn(b._h, x_ptr, MAX_IN, lp, y_ptr, cap, cap, cp)
            else:
                fn = L.r8bgpu_batch_process_host_ragged_fmt if host else L.r8bgpu_batch_process_ragged_fmt
                rc = fn(b._h, C.byref(bi), lp, C.byref(bo), cap, cp)
            if rc < 0:
                raise pkg.R8bGpuError(pkg._err())
            n_out[0] += int(counts.sum())
            return int(lens_c[i].sum())
        b.process_ptr(x.data_ptr(), MAX_IN, mean_len, y.data_ptr(), cap, cap)
        return mean_len * n_ch

    for i in range(warmup):
        call(i % len(lens_c))
    torch.cuda.synchronize()
    l0 = b.kernel_launches
    n_out[0] = 0
    t0 = time.perf_counter()
    n_in = 0
    for i in range(warmup, len(lens_c)):
        n_in += call(i)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    steps = len(lens_c) - warmup
    r = {"src": src, "dst": dst, "channels": n_ch,
         "mode": "ragged" if ragged else "lockstep, unfused" if unfused else "lockstep",
         "form": "host" if host else "device", "format": fmt,
         "block_len": "%d..%d" % (int(np.min(lens_seq)), int(np.max(lens_seq))) if ragged else mean_len,
         "in_samples_per_s": n_in / dt, "ms_per_call": 1e3 * dt / steps,
         "launches_per_call": (b.kernel_launches - l0) / steps}
    if host:  # the samples that cross PCIe: each block in, each channel's count out
        r["pcie_bytes_per_in_sample"] = esize * (n_in + n_out[0]) / n_in
        pkg.host_free(x)
        pkg.host_free(y)
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--channels", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--min-len", type=int, default=32768)
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--format", default="f64", choices=sorted(FORMATS), help="sample format of the ragged calls' buffers")
    ap.add_argument("--host", action="store_true", help="ragged calls through the host form, on pinned host buffers")
    args = ap.parse_args()
    import torch
    from __graft_entry__ import load_package
    pkg = load_package()
    if not torch.cuda.is_available():
        raise SystemExit("ragged_bench: no CUDA device")
    rng = np.random.default_rng(args.seed)
    lens_seq = rng.integers(args.min_len, MAX_IN + 1, size=(args.warmup + args.steps, args.channels))
    gpu = torch.cuda.get_device_name(0)
    q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    power = q.stdout.strip() if q.returncode == 0 else "unknown"
    modes = ((False, False), (False, True), (True, False))
    if args.host or args.format != "f64":
        modes = ((True, False),)
    for src, dst in CASES:
        for ragged, unfused in modes:
            r = run(pkg, torch, src, dst, args.channels, lens_seq, ragged, args.warmup, unfused, args.format, args.host)
            r["gpu"] = gpu
            r["power_limit"] = power
            print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
