"""Cost of drift compensation on same-rate and integer-ratio links: trim plans for any rate pair (Plan.asrc) at
48000->48000 and 44100->88200, next to an ordinary ragged plan of a rate a little off 48000.

Each case is one batch of --channels channels (default 1024), CDSPResampler24, max_trim 2e-4.  Two block regimes: long
blocks (lengths drawn per channel and call from [8192, 16384], MaxInLen 16384) and live blocks ([441, 882], MaxInLen
882, 10 to 20 ms of audio).  Every mode of a regime feeds the same ragged block lengths, drawn with a fixed seed, from
device buffers on one stream:
  drift   asrc plan; before every call each channel's factor takes a step of a random walk within +-200 ppm
          (Batch.set_trim), so every channel runs on its own schedule
  unit    the same asrc plan with every factor 1
  ragged  for reference: the ordinary 48000->47999 plan, r8bgpu_batch_process_ragged
The modes alternate --rounds times; each run times --steps calls after --warmup calls with CUDA events around the calls
and a host clock around the same window ending in a device synchronise (the host clock includes the host-side planning
of every call).  Prints one JSON line per regime, case and mode with the median over the rounds and the GPU's name and
power limit."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from trim_bench import gpu_info, run  # noqa: E402

MAX_TRIM = 2e-4
REGIMES = {"long": (8192, 16384), "live": (441, 882)}
# (case, mode): the plan each run builds
RUNS = [((48000.0, 48000.0), "drift"), ((48000.0, 48000.0), "unit"), ((44100.0, 88200.0), "drift"),
        ((44100.0, 88200.0), "unit"), ((48000.0, 47999.0), "ragged")]


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--channels", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=6)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--regimes", default="long,live")
    a = ap.parse_args()
    import torch
    import __graft_entry__
    pkg = __graft_entry__.load_package()
    if not torch.cuda.is_available() or pkg.device_count() < 1:
        raise SystemExit("asrc_bench: no CUDA device")
    gpu = gpu_info()
    for regime in a.regimes.split(","):
        lo, max_in = REGIMES[regime]
        rng = np.random.default_rng(1)
        lens_seq = [np.ascontiguousarray(rng.integers(lo, max_in + 1, a.channels), dtype=np.int32)
                    for _ in range(a.warmup + a.steps)]
        res = {r: [] for r in RUNS}
        for _ in range(a.rounds):
            for (src, dst), m in RUNS:
                plan = pkg.Plan(src, dst, max_in, 2.0, pkg.ATTEN_24) if m == "ragged" else \
                    pkg.Plan.asrc(src, dst, max_in, 2.0, pkg.ATTEN_24, MAX_TRIM)
                res[((src, dst), m)].append(run(pkg, torch, plan, m, a.channels, max_in, lens_seq, a.warmup, a.steps))
        for ((src, dst), m), rs in res.items():
            med = {k: float(np.median([r[k] for r in rs])) for k in rs[0]}
            med["ms_per_call_wall_all"] = [round(r["ms_per_call_wall"], 4) for r in rs]
            print(json.dumps(dict(regime=regime, case="%g->%g" % (src, dst), mode=m, channels=a.channels, max_in=max_in,
                                  gpu=gpu, **med)), flush=True)


if __name__ == "__main__":
    main()
