"""DSD output against fp64 output on the same input: lock-step calls, the arms alternated --rounds times.

  dsd64_44k    512 channels 44100->2822400  (the 64x half-band up-cascade)
  dsd64_48k   1024 channels 48000->3072000
  dsd256_44k   256 channels 44100->11289600
Arms: F64 (planar doubles) and DSD_LSB planar (r8bgpu_batch_set_dsd_out), scale 0.5, on a PCM mix of sines and noise.
  device   device-resident buffers (r8bgpu_batch_process_fmt), ms per call from CUDA events over --steps calls after
           --warmup calls;
  host     pinned host buffers (r8bgpu_batch_process_host_fmt, every call synchronises), ms per call by host clock, and
           G input samples/s.
Then, in a run of its own with the batch's stage timing on, K8's (k_dsd_mod's) own device time per DSD call from the
CUDA events around its launches (r8bgpu_batch_stage_time_ms, the stage after the plan's last), and that over the samples
one channel walks: the walk's time per sample (every channel walks at once).  Before timing, one call of each arm from a
fresh batch must give DSD bytes equal to the host modulator's on the F64 arm's outputs (else the run stops).  One JSON line per
case, arm and path, with the GPU's name, power limit and max SM clock read by a read-only nvidia-smi query in the same
run."""
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

CASES = [("dsd64_44k", 512, 44100.0, 2822400.0, 4096), ("dsd64_48k", 1024, 48000.0, 3072000.0, 4096),
         ("dsd256_44k", 256, 44100.0, 11289600.0, 4096)]
ARMS = ["F64", "DSD"]
SCALE = 0.5


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
        raise SystemExit("dsd_out_bench: no CUDA device visible")
    info = gpu_info()
    for name, nch, src, dst, L in CASES:
        if name not in a.cases.split(","):
            continue
        plan = P.Plan(src, dst, L, 2.0, P.ATTEN_24)
        cap = plan.max_out_len
        cap8 = (cap + 7) // 8 * 8
        t = np.arange(L)
        x = 0.8 * np.sin(2 * np.pi * 997.0 / src * (t[None, :] + 311 * np.arange(nch)[:, None]))
        x += 0.05 * np.random.default_rng(1).standard_normal((nch, L))
        d_in = torch.from_numpy(x).cuda()
        d_out = {"F64": torch.zeros((nch, cap), dtype=torch.float64, device="cuda"),
                 "DSD": torch.zeros((nch, cap8 // 8), dtype=torch.uint8, device="cuda")}
        bi_d = P.Buffer.make(d_in.data_ptr(), P.F64, False, L, 1.0)
        bo_d = {"F64": P.Buffer.make(d_out["F64"].data_ptr(), P.F64, False, cap, 1.0),
                "DSD": P.Buffer.make(d_out["DSD"].data_ptr(), P.DSD_LSB, False, cap8 // 8, SCALE)}

        def batch(arm):
            b = P.Batch(plan, nch)
            if arm == "DSD":
                b.set_dsd_out(True)
            b.set_stream(torch.cuda.current_stream().cuda_stream)
            return b

        def dev_call(b, arm):
            return b.process_fmt(bi_d, L, bo_d[arm], cap8 if arm == "DSD" else cap, host=False)

        # the DSD arm's bytes against the host modulator on the F64 arm's outputs (a few channels)
        b = batch("F64")
        n = dev_call(b, "F64")
        y = d_out["F64"][:, :n].cpu().numpy()
        del b
        b = batch("DSD")
        nb = dev_call(b, "DSD")
        got = d_out["DSD"][:, :nb // 8].cpu().numpy()
        del b
        for c in (0, 1, 31, 32, nch // 2, nch - 1):
            want = np.packbits(P.dsd_modulate(y[c], SCALE)[0][:nb], bitorder="little")
            assert np.array_equal(got[c], want), "%s: DSD bytes of channel %d differ from the host modulator's" % (name, c)
        # host arms: pinned buffers
        hb = P.Batch(plan, nch)
        h_in = hb.host_alloc(L, "float64")
        h_in[:] = x
        h_out = {"F64": hb.host_alloc(cap, "float64"), "DSD": hb.host_alloc(cap8 // 8, "uint8")}
        bi_h = P.Buffer.make(h_in.ctypes.data, P.F64, False, L, 1.0)
        bo_h = {"F64": P.Buffer.make(h_out["F64"].ctypes.data, P.F64, False, cap, 1.0),
                "DSD": P.Buffer.make(h_out["DSD"].ctypes.data, P.DSD_LSB, False, cap8 // 8, SCALE)}
        res = {}
        for _ in range(a.rounds):
            for arm in ARMS:
                b = batch(arm)
                for _ in range(a.warmup):
                    dev_call(b, arm)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(a.steps):
                    dev_call(b, arm)
                e1.record()
                torch.cuda.synchronize()
                res.setdefault((arm, "device"), []).append(e0.elapsed_time(e1) / a.steps)
                del b
                b = batch(arm)
                oc = cap8 if arm == "DSD" else cap
                for _ in range(a.warmup):
                    b.process_fmt(bi_h, L, bo_h[arm], oc, host=True)
                t0 = time.perf_counter()
                for _ in range(a.steps):
                    b.process_fmt(bi_h, L, bo_h[arm], oc, host=True)
                res.setdefault((arm, "host"), []).append((time.perf_counter() - t0) * 1e3 / a.steps)
                del b
        # K8's own device time: CUDA events around its launches, in a run of its own
        b = batch("DSD")
        for _ in range(a.warmup):
            dev_call(b, "DSD")
        b.set_timing(True)
        for _ in range(a.steps):
            dev_call(b, "DSD")
        k8_launches = C.c_ulonglong(0)
        k8_ms = P.lib().r8bgpu_batch_stage_time_ms(b._h, len(plan.stages()), C.byref(k8_launches))
        assert k8_ms >= 0 and k8_launches.value == a.steps, (k8_ms, k8_launches.value)
        k8_us = k8_ms * 1e3 / a.steps
        del b
        for arm in ARMS:
            for path in ("device", "host"):
                v = res[(arm, path)]
                ms = float(np.median(v))
                rec = {"case": name, "arm": arm, "path": path, "channels": nch, "src": src, "dst": dst, "block": L,
                       "outputs_per_channel": n, "ms_per_call_median": round(ms, 4), "ms_all_rounds": [round(t, 4) for t in v],
                       "g_in_samples_per_s": round(nch * L / (ms * 1e-3) / 1e9, 3), "gpu": info}
                if arm == "DSD" and path == "device":
                    rec["k_dsd_mod_ms"] = round(k8_us / 1e3, 4)
                    rec["walk_ns_per_sample"] = round(k8_us * 1e3 / n, 3)
                print(json.dumps(rec), flush=True)
        P.host_free(h_in)
        P.host_free(h_out["F64"])
        P.host_free(h_out["DSD"])
        del d_in, d_out, hb


if __name__ == "__main__":
    main()
