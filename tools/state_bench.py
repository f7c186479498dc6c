"""Cost of moving streams: export and import of 1024 channels, host and device forms (Batch.export_channels /
import_channels over r8bgpu_batch_export / _import / _export_device / _import_device).

Each batch first runs a few diverged ragged calls, so every ring holds real history; then each form is timed over
--reps calls (wall clock around the synchronising call).  Prints one JSON line per (rate pair, form, direction) with
ms per call, bytes per channel, and the board it ran on.

    python tools/state_bench.py [--channels 1024] [--max-in 65536] [--reps 5]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--channels", type=int, default=1024)
    ap.add_argument("--max-in", type=int, default=65536)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    import __graft_entry__
    import torch
    pkg = __graft_entry__.load_package()
    n, M = a.channels, a.max_in
    board = torch.cuda.get_device_name(0)
    ch = np.arange(n, dtype=np.int32)
    for src, dst in ((44100.0, 96000.0), (48000.0, 44100.0)):
        plan = pkg.Plan(src, dst, M, 2.0, 180.15)
        A = pkg.Batch(plan, n, 0)
        B = pkg.Batch(plan, n, 0)
        rng = np.random.default_rng(1)
        for _ in range(3):
            lens = rng.integers(M // 2, M + 1, size=n)
            x = torch.randn(n, M, dtype=torch.float64, device="cuda")
            A.process_ragged([x[c, :lens[c]] for c in range(n)])
        torch.cuda.synchronize()
        for form in ("host", "device"):
            dev = form == "device"
            blobs = A.export_channels(ch, device=dev)  # warm-up: staging, link rings
            B.import_channels(ch, blobs)
            for what, fn in (("export", lambda: A.export_channels(ch, device=dev)),
                             ("import", lambda: B.import_channels(ch, blobs))):
                ts = []
                for _ in range(a.reps):
                    torch.cuda.synchronize()
                    t = time.perf_counter()
                    fn()
                    torch.cuda.synchronize()
                    ts.append((time.perf_counter() - t) * 1e3)
                print(json.dumps({"pair": "%g->%g" % (src, dst), "form": form, "op": what, "channels": n, "max_in_len": M,
                                  "ms_per_call_median": round(float(np.median(ts)), 3),
                                  "ms_per_call_min": round(float(np.min(ts)), 3),
                                  "bytes_per_channel": plan.state_bytes, "board": board}), flush=True)


if __name__ == "__main__":
    main()
