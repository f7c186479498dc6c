"""Long clips at mixed rates: one Batch.oneshot_long / oneshot_adjoint call with plan_of on a mixed batch, against one
ordinary batch per rate called in turn, on a dataset-like batch:

  512 clips of 2-30 s (uniform), a quarter each at 16000, 22050, 44100 and 48000 Hz, all going to 16000 Hz (the 16000
  part is a passthrough), float32 CUDA tensors, MaxInLen 65536, CDSPResampler24; lanes split across the parts
  (default 64 / 192 / 384 / 384 of 1024).

Arms, forward and adjoint:
  (a) mixed     one call with plan_of on the mixed batch;
  (b) per-rate  one ordinary batch per rate with the same lanes, called in sequence on one stream; the caller's split
                (index_select of its rows) and merge (index_copy_ into one padded output) are inside the timed region;
  (c) clips     forward only: Batch.oneshot_clips on the mixed batch, one clip per channel, so only as many clips of a
                rate as its part has channels (the first ones of each rate).

Every arm finishes before it returns; times are CUDA events around each call on torch's current stream, after one
warm-up call of each arm, the arms alternating over --reps repetitions.  The best and the median of each arm are
printed, with the input samples per second and the GPU's name, power limit and max SM clock.  The run stops unless the
arms' outputs are bit-identical (clip by clip; arm (c) on its clips)."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from __graft_entry__ import load_package  # noqa: E402

RATES = [16000.0, 22050.0, 44100.0, 48000.0]
DST = 16000.0


def gpu_line():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # the numbers still stand; say what is missing
        return "unknown (%s)" % e


def timed(torch, f):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out = f()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clips", type=int, default=512)
    ap.add_argument("--min-s", type=float, default=2.0)
    ap.add_argument("--max-s", type=float, default=30.0)
    ap.add_argument("--lanes", default="64,192,384,384", help="lanes of the 16000/22050/44100/48000 parts")
    ap.add_argument("--max-in", type=int, default=65536)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    import torch
    pkg = load_package()
    gpu = gpu_line()
    lanes = [int(v) for v in a.lanes.split(",")]
    plans = [pkg.Plan(s, DST, a.max_in, 2.0, pkg.ATTEN_24) for s in RATES]
    rng = np.random.default_rng(7)
    po = np.arange(a.clips, dtype=np.int32) % len(RATES)
    rng.shuffle(po)
    lens = np.array([int(RATES[p] * rng.uniform(a.min_s, a.max_s)) for p in po], dtype=np.int64)
    chan_plan = np.concatenate([np.full(n, p, np.int32) for p, n in enumerate(lanes)])
    mb = pkg.Batch.mixed(plans, chan_plan, device=0)
    ob = [pkg.Batch(plans[p], lanes[p], device=0) for p in range(len(RATES))]
    rows = [torch.from_numpy(np.nonzero(po == p)[0]).cuda() for p in range(len(RATES))]
    gen = torch.Generator(device="cuda").manual_seed(1)
    x = torch.rand((a.clips, int(lens.max())), dtype=torch.float32, device="cuda", generator=gen) * 2 - 1
    x *= torch.arange(x.shape[1], device="cuda")[None, :] < torch.from_numpy(lens).cuda()[:, None]

    def mixed_fwd():
        return mb.oneshot_long(x, lens, plan_of=po)[0]

    def split_fwd():
        y = torch.zeros(mixed_y.shape, dtype=torch.float32, device="cuda")
        for p in range(len(RATES)):
            lp = lens[po == p]
            yp, _ = ob[p].oneshot_long(x.index_select(0, rows[p])[:, :int(lp.max())], lp)
            y[:, :yp.shape[1]].index_copy_(0, rows[p], yp)
        return y

    # arm (c): for each channel of the mixed batch the next clip of its plan, while there is one
    pick = -np.ones(len(chan_plan), dtype=np.int64)
    for p in range(len(RATES)):
        ch, cl = np.nonzero(chan_plan == p)[0], np.nonzero(po == p)[0]
        k = min(len(ch), len(cl))
        pick[ch[:k]] = cl[:k]
    lens_c = np.where(pick >= 0, lens[np.maximum(pick, 0)], 0)
    op_c = np.array([plans[chan_plan[c]].default_target(int(lens_c[c])) for c in range(len(chan_plan))], dtype=np.int64)
    xc = x.index_select(0, torch.from_numpy(np.maximum(pick, 0)).cuda())[:, :int(lens_c.max())].contiguous()
    xc *= torch.from_numpy(pick >= 0).cuda()[:, None]

    def clips_fwd():
        return mb.oneshot_clips(xc, lens_c, op_c)[0]

    mixed_y = mixed_fwd()
    oplens = np.array([plans[p].default_target(int(n)) for p, n in zip(po, lens)], dtype=np.int64)
    g = torch.rand(mixed_y.shape, dtype=torch.float32, device="cuda", generator=gen) * 2 - 1
    g *= torch.arange(g.shape[1], device="cuda")[None, :] < torch.from_numpy(oplens).cuda()[:, None]

    def mixed_adj():
        return mb.oneshot_adjoint(g, lens, oplens, width=x.shape[1], plan_of=po)

    def split_adj():
        gx = torch.zeros(x.shape, dtype=torch.float32, device="cuda")
        for p in range(len(RATES)):
            lp, op = lens[po == p], oplens[po == p]
            gp = ob[p].oneshot_adjoint(g.index_select(0, rows[p])[:, :int(op.max())], lp, op, width=int(lp.max()))
            gx[:, :gp.shape[1]].index_copy_(0, rows[p], gp)
        return gx

    # the arms must agree bit for bit
    if not torch.equal(mixed_y, split_fwd()):
        sys.exit("forward: the mixed call and the per-rate calls differ")
    yc = clips_fwd()
    for c in np.nonzero(pick >= 0)[0]:
        if not torch.equal(yc[c, :op_c[c]], mixed_y[pick[c], :op_c[c]]):
            sys.exit("forward: oneshot_clips differs from the mixed call on clip %d" % pick[c])
    if not torch.equal(mixed_adj(), split_adj()):
        sys.exit("adjoint: the mixed call and the per-rate calls differ")
    arms = {"fwd_mixed": mixed_fwd, "fwd_per_rate": split_fwd, "fwd_clips": clips_fwd,
            "adj_mixed": mixed_adj, "adj_per_rate": split_adj}
    ms = {k: [] for k in arms}
    for _ in range(a.reps):
        for k, f in arms.items():
            ms[k].append(timed(torch, f)[0])
    samples = float(lens.sum())
    res = {"clips": a.clips, "seconds": [a.min_s, a.max_s], "rates": RATES, "dst": DST, "lanes": lanes, "max_in": a.max_in,
           "input_samples": int(samples), "clips_arm_clips": int((pick >= 0).sum()), "gpu": gpu}
    for k in arms:
        res[k + "_ms"] = {"best": round(min(ms[k]), 2), "median": round(float(np.median(ms[k])), 2)}
        if k != "fwd_clips":
            res[k + "_msamples_per_s"] = round(samples / min(ms[k]) / 1e3, 1)
    res["fwd_clips_msamples_per_s"] = round(float(lens_c.sum()) / min(ms["fwd_clips"]) / 1e3, 1)
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
