"""DSD input against fp64 input on the same bits: lock-step calls, the arms alternated --rounds times.

  dsd64_44k   1024 channels  2822400->44100  (CDSPResampler24; bench.py's cfg3c chain)
  dsd64_48k   1024 channels  2822400->48000
  dsd256_44k   256 channels 11289600->44100
Arms: F64 (planar doubles, +-1.0 per bit), DSD_LSB planar, DSD_LSB interleaved (DSDIFF's byte interleave).
  device   device-resident buffers (r8bgpu_batch_process / _fmt), ms per call from CUDA events over --steps calls after
           --warmup calls, and kernel launches per call;
  host     pinned host buffers (r8bgpu_batch_process_host_fmt, every call synchronises), ms per call by host clock.
Before timing, one call of each arm from a fresh batch on the same bits checks that the DSD arms' outputs equal the F64
arm's bit for bit.  One JSON line per case, arm and path, with the GPU's name, power limit and max SM clock read by a
read-only nvidia-smi query in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CASES = [("dsd64_44k", 1024, 2822400.0, 44100.0, 65536), ("dsd64_48k", 1024, 2822400.0, 48000.0, 65536),
         ("dsd256_44k", 256, 11289600.0, 44100.0, 262144)]
ARMS = ["F64", "DSD_planar", "DSD_interleaved"]


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
    import torch

    import __graft_entry__
    P = __graft_entry__.load_package()
    if P.device_count() < 1:
        raise SystemExit("dsd_bench: no CUDA device visible")
    info = gpu_info()
    rng = np.random.default_rng(1)
    for name, nch, src, dst, L in CASES:
        if name not in a.cases.split(","):
            continue
        plan = P.Plan(src, dst, L, 2.0, P.ATTEN_24)
        cap = plan.max_out_len
        bits = rng.integers(0, 256, (nch, L // 8)).astype(np.uint8)
        planar = bits
        inter = np.ascontiguousarray(bits.T)
        f64 = np.where(np.unpackbits(bits, axis=1, bitorder="little") != 0, 1.0, -1.0)
        d_in = {"F64": torch.from_numpy(f64).cuda(), "DSD_planar": torch.from_numpy(planar).cuda(),
                "DSD_interleaved": torch.from_numpy(inter).cuda()}
        d_out = torch.zeros((nch, cap), dtype=torch.float64, device="cuda")

        def buf_in(arm, ptr):
            if arm == "F64":
                return P.Buffer.make(ptr, P.F64, False, L, 1.0)
            return P.Buffer.make(ptr, P.DSD_LSB, arm == "DSD_interleaved", nch if arm == "DSD_interleaved" else L // 8, 1.0)

        def dev_call(b, arm):
            b.process_fmt(buf_in(arm, d_in[arm].data_ptr()), L, P.Buffer.make(d_out.data_ptr(), P.F64, False, cap), cap,
                          host=False)

        # bit-identity of the arms: one call each from a fresh batch
        first = {}
        for arm in ARMS:
            b = P.Batch(plan, nch)
            b.set_stream(torch.cuda.current_stream().cuda_stream)
            dev_call(b, arm)
            torch.cuda.synchronize()
            first[arm] = d_out.cpu().numpy().copy()
            del b
        identical = all(np.array_equal(first[arm], first["F64"]) for arm in ARMS)
        # host arms: pinned buffers
        hb = P.Batch(plan, nch)
        h_in = {"F64": hb.host_alloc(L, "float64"), "DSD_planar": hb.host_alloc(L // 8, "uint8")}
        h_in["F64"][:] = f64
        h_in["DSD_planar"][:] = planar
        h_il = hb.host_alloc(L // 8, "uint8")  # pinned bytes, used as [L / 8 byte frames][nch]
        h_il.reshape(L // 8, nch)[:] = inter
        h_out = hb.host_alloc(cap, "float64")
        bo_h = P.Buffer.make(h_out.ctypes.data, P.F64, False, cap, 1.0)
        res = {}
        for _ in range(a.rounds):
            for arm in ARMS:
                b = P.Batch(plan, nch)
                b.set_stream(torch.cuda.current_stream().cuda_stream)
                for _ in range(a.warmup):
                    dev_call(b, arm)
                n0 = b.kernel_launches
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(a.steps):
                    dev_call(b, arm)
                e1.record()
                torch.cuda.synchronize()
                res.setdefault((arm, "device"), []).append(e0.elapsed_time(e1) / a.steps)
                res[(arm, "launches")] = (b.kernel_launches - n0) / a.steps
                del b
                if arm == "DSD_interleaved":
                    bi = P.Buffer.make(h_il.ctypes.data, P.DSD_LSB, True, nch, 1.0)
                else:
                    bi = buf_in(arm, h_in[arm].ctypes.data)
                b = P.Batch(plan, nch)
                for _ in range(a.warmup):
                    b.process_fmt(bi, L, bo_h, cap, host=True)
                t = time.perf_counter()
                for _ in range(a.steps):
                    b.process_fmt(bi, L, bo_h, cap, host=True)
                res.setdefault((arm, "host"), []).append((time.perf_counter() - t) * 1e3 / a.steps)
                del b
        for arm in ARMS:
            for path in ("device", "host"):
                v = res.get((arm, path))
                if not v:
                    continue
                ms = float(np.median(v))
                print(json.dumps({"case": name, "arm": arm, "path": path, "channels": nch, "src": src, "dst": dst, "block": L,
                                  "ms_per_call_median": round(ms, 4), "ms_all_rounds": [round(t, 4) for t in v],
                                  "g_in_samples_per_s": round(nch * L / (ms * 1e-3) / 1e9, 3),
                                  "launches_per_call": res[(arm, "launches")], "outputs_identical_to_f64": identical,
                                  "gpu": info}), flush=True)
        P.host_free(h_in["F64"])
        P.host_free(h_in["DSD_planar"])
        P.host_free(h_il)
        P.host_free(h_out)
        del d_in, d_out, hb


if __name__ == "__main__":
    main()
