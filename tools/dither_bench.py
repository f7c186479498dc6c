"""Cost of dithered int16 output: OFF (the plain cast), flat TPDF and 9-tap noise shaping on 1024 channels.

  cfg2    44100->96000, CDSPResampler24, 65536-sample blocks, lock-step typed calls: device-resident
          (r8bgpu_batch_process_fmt, fp64 in, int16 out) and end to end from host buffers (_process_host_fmt)
  live    48000->44100, ragged typed calls of 441..882 samples per channel (seeded), device-resident
Every mode runs --warmup calls, then --steps calls timed with CUDA events around the window (device) or a host clock
around calls that synchronise (host); the modes alternate --rounds times and each prints its median with the GPU's name
and power limit, one JSON line per case and mode."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

TAPS9 = [2.033, -2.165, 1.959, -1.590, 0.6149, -0.2, 0.1, -0.05, 0.01]
MODES = {"off": None, "tpdf": [], "shaped9": TAPS9}


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0] if r.stdout.strip() else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--channels", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    import torch
    import __graft_entry__
    P = __graft_entry__.load_package()
    info = gpu_info()
    nch = a.channels
    ch = np.arange(nch)

    def batch(plan, mode):
        b = P.Batch(plan, nch)
        if MODES[mode] is not None:
            b.set_dither(ch, ch + 1, MODES[mode])
        b.set_stream(torch.cuda.current_stream().cuda_stream)
        return b

    def timed_dev(fn):
        for _ in range(a.warmup):
            fn()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(a.steps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / a.steps

    def timed_host(fn):
        for _ in range(a.warmup):
            fn()
        t = time.perf_counter()
        for _ in range(a.steps):
            fn()
        return (time.perf_counter() - t) * 1e3 / a.steps

    # cfg 2
    L = 65536
    plan2 = P.Plan(44100.0, 96000.0, L, 2.0, P.ATTEN_24)
    cap = plan2.max_out_len
    x = (0.5 * torch.randn(nch, L, dtype=torch.float64, device="cuda")).clamp_(-1, 1)
    y = torch.zeros(nch, cap, dtype=torch.int16, device="cuda")
    hx = np.ascontiguousarray(x.cpu().numpy())
    hy = np.zeros((nch, cap), np.int16)
    bi = P.Buffer.make(x.data_ptr(), P.F64, False, L)
    bo = P.Buffer.make(y.data_ptr(), P.S16, False, cap, 32767.0)
    hbi = P.Buffer.make(hx.ctypes.data, P.F64, False, L)
    hbo = P.Buffer.make(hy.ctypes.data, P.S16, False, cap, 32767.0)
    # live-sized ragged calls
    plan_l = P.Plan(48000.0, 44100.0, 882, 2.0, P.ATTEN_24)
    lens = np.random.default_rng(1).integers(441, 883, nch).astype(np.int32)
    xl = (0.5 * torch.randn(nch, 882, dtype=torch.float64, device="cuda")).clamp_(-1, 1)
    res = {}
    for _ in range(a.rounds):
        for mode in MODES:
            b = batch(plan2, mode)
            res.setdefault(("cfg2_device", mode), []).append(timed_dev(lambda: b.process_fmt(bi, L, bo, cap, host=False)))
            res.setdefault(("cfg2_host", mode), []).append(timed_host(lambda: b.process_fmt(hbi, L, hbo, cap, host=True)))
            del b
            bl = batch(plan_l, mode)
            res.setdefault(("live_ragged", mode), []).append(
                timed_dev(lambda: bl.process_ragged_fmt(xl, lens, out_fmt=P.S16, out_scale=32767.0)))
            del bl
    for (case, mode), v in res.items():
        print(json.dumps({"case": case, "mode": mode, "channels": nch, "ms_per_call_median": float(np.median(v)),
                          "ms_all_rounds": [round(t, 4) for t in v], "gpu": info}))


if __name__ == "__main__":
    main()
