"""End-to-end host-buffer rate of one-byte samples against int16: lock-step typed calls (r8bgpu_batch_process_host_fmt)
from pinned planar host buffers, the same shape for each format, the formats alternated --rounds times.

  tel_up    4096 channels  8000->16000, int16 vs G.711 mu-law in and out
  tel_down  4096 channels 16000->8000,  int16 vs G.711 mu-law in and out
  cfg2      1024 channels 44100->96000 (CDSPResampler24), int16 vs unsigned 8-bit in and out
Each case runs --warmup calls, then --steps calls timed with a host clock (every call synchronises).  One JSON line per
case and format: the median time per call, input samples per second, the PCIe bytes per input sample (computed: in +
out * dst/src), and the GPU's name, power limit and max SM clock."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CASES = [("tel_up", 4096, 8000.0, 16000.0, 16384, "ULAW"), ("tel_down", 4096, 16000.0, 8000.0, 16384, "ULAW"),
         ("cfg2", 1024, 44100.0, 96000.0, 65536, "U8")]


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0] if r.stdout.strip() else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--cases", default=",".join(c[0] for c in CASES))
    a = ap.parse_args()
    import __graft_entry__
    P = __graft_entry__.load_package()
    if P.device_count() < 1:
        raise SystemExit("g711_bench: no CUDA device visible")
    info = gpu_info()
    rng = np.random.default_rng(1)
    for name, nch, src, dst, L, narrow in CASES:
        if name not in a.cases.split(","):
            continue
        plan = P.Plan(src, dst, L, 2.0, P.ATTEN_24)
        cap = plan.max_out_len
        fmts = {"S16": (P.S16, "int16", 1.0 / 32768, 32767.0), narrow: (getattr(P, narrow), "uint8",
                                                                      1.0 / 128 if narrow == "U8" else 1.0 / 32768,
                                                                      127.0 if narrow == "U8" else 32767.0)}
        runs = {}
        for key, (fmt, dt, isc, osc) in fmts.items():
            b = P.Batch(plan, nch)
            hx, hy = b.host_alloc(L, dt), b.host_alloc(cap, dt)
            hx[:] = rng.integers(np.iinfo(dt).min // 2, np.iinfo(dt).max // 2, hx.shape).astype(dt)
            bi = P.Buffer.make(hx.ctypes.data, fmt, False, L, isc)
            bo = P.Buffer.make(hy.ctypes.data, fmt, False, cap, osc)
            runs[key] = (b, hx, hy, bi, bo)
        res = {k: [] for k in fmts}
        for _ in range(a.rounds):
            for key, (b, hx, hy, bi, bo) in runs.items():
                for _ in range(a.warmup):
                    b.process_fmt(bi, L, bo, cap, host=True)
                t = time.perf_counter()
                for _ in range(a.steps):
                    b.process_fmt(bi, L, bo, cap, host=True)
                res[key].append((time.perf_counter() - t) * 1e3 / a.steps)
        for key, v in res.items():
            e = P.FORMAT_BYTES[fmts[key][0]]
            ms = float(np.median(v))
            print(json.dumps({"case": name, "format": key, "channels": nch, "src": src, "dst": dst, "block": L,
                              "ms_per_call_median": round(ms, 4), "ms_all_rounds": [round(t, 4) for t in v],
                              "g_in_samples_per_s": round(nch * L / (ms * 1e-3) / 1e9, 3),
                              "pcie_bytes_per_in_sample": round(e + e * dst / src, 3), "gpu": info}), flush=True)
        for b, hx, hy, _, _ in runs.values():
            P.host_free(hx)
            P.host_free(hy)
        del runs


if __name__ == "__main__":
    main()
