"""Throughput of a mixed batch (r8bgpu_batch_create_mixed): independent streams at different source rates in one batch,
next to what a caller without one does.

--channels channels (default 1024) with source rates drawn from {16000, 22050, 32000, 44100, 48000, 96000} (seeded),
all to 48000 (48000 -> 48000 is a passthrough plan), MaxInLen 65536, ragged block lengths drawn from [--min-len, 65536].
Cases:
  mixed    one mixed batch; every call is one ragged call on it
  buckets  one ordinary batch per source rate, called one after another on one stream, with the rows gathered out of
           the caller's buffer (torch index_select) before each bucket's call and its outputs scattered back into
           per-channel order (index_copy_) after it -- what a caller had to do without mixed batches
Formats f64 and s16 (--formats), device buffers and the host form (pinned buffers, copies inside the timed region).
Timed with a device synchronise around --steps calls after --warmup calls.  One JSON line per case: input samples per
second over all channels (G/s), ms per call and kernel launches per call, with the card name and power limit.

--cases mixed --label NAME runs only the mixed case and tags its lines (for experiment builds loaded through
R8BGPU_LIB_PATH).  --profile adds one torch.profiler pass over mixed device calls and reports the mapped conversions'
share of the kernel time.  Sampled channels of a fresh mixed batch are checked against the reference (oracle/_ref),
when it is built."""
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
sys.path.insert(0, os.path.join(ROOT, "tests"))

RATES = [16000.0, 22050.0, 32000.0, 44100.0, 48000.0, 96000.0]
DST = 48000.0
MAX_IN = 65536
FORMATS = {"f64": ("float64", 0), "s16": ("int16", 2)}


class Setup:
    def __init__(self, pkg, torch, n_ch, seed):
        rng = np.random.default_rng(seed)
        self.plan_of = rng.integers(0, len(RATES), size=n_ch).astype(np.int32)
        self.plan_of[:len(RATES)] = np.arange(len(RATES))
        self.plans = [pkg.Plan(s, DST, MAX_IN, 2.0, pkg.ATTEN_24) for s in RATES]
        self.rows = [np.nonzero(self.plan_of == p)[0] for p in range(len(RATES))]
        self.n_ch = n_ch


def run(pkg, torch, S, case, fmt, host, lens_seq, warmup):
    L = pkg.lib()
    n_ch = S.n_ch
    dtype, code = FORMATS[fmt]
    tdt = getattr(torch, dtype)
    amp = 20000.0 if fmt == "s16" else 1.0
    dev = "cpu" if host else "cuda:0"
    x = ((torch.rand((n_ch, MAX_IN), dtype=torch.float64, device=dev) * 2 - 1) * amp).to(tdt)
    counts = np.empty(n_ch, dtype=np.int32)
    lens_c = [np.ascontiguousarray(v, dtype=np.int32) for v in lens_seq]
    stream = torch.cuda.current_stream().cuda_stream
    if case == "mixed":
        b = pkg.Batch.mixed(S.plans, S.plan_of, 0)
        b.set_stream(stream)
        cap = b.max_out_len
        y = torch.empty((n_ch, cap), dtype=tdt, device=dev)
        if host:
            x, y = x.pin_memory(), y.pin_memory()
        bi, bo = pkg.Buffer.make(x.data_ptr(), code, False, MAX_IN), pkg.Buffer.make(y.data_ptr(), code, False, cap)
        fn = L.r8bgpu_batch_process_host_ragged_fmt if host else L.r8bgpu_batch_process_ragged_fmt
        batches = [b]

        def call(lens):
            if fn(b._h, C.byref(bi), lens.ctypes.data, C.byref(bo), cap, counts.ctypes.data) < 0:
                raise pkg.R8bGpuError(pkg._err())
    else:
        bs = [pkg.Batch(p, len(r), 0) for p, r in zip(S.plans, S.rows)]
        for b in bs:
            b.set_stream(stream)
        cap = max(p.max_out_len for p in S.plans)
        y = torch.empty((n_ch, cap), dtype=tdt, device=dev)
        idx = [torch.as_tensor(r, device=dev) for r in S.rows]
        caps = [p.max_out_len for p in S.plans]
        xb = [torch.empty((len(r), MAX_IN), dtype=tdt, device=dev) for r in S.rows]
        yb = [torch.empty((len(r), c), dtype=tdt, device=dev) for r, c in zip(S.rows, caps)]
        if host:
            xb, yb = [t.pin_memory() for t in xb], [t.pin_memory() for t in yb]
        fn = L.r8bgpu_batch_process_host_ragged_fmt if host else L.r8bgpu_batch_process_ragged_fmt
        bufs = [(pkg.Buffer.make(a.data_ptr(), code, False, MAX_IN), pkg.Buffer.make(o.data_ptr(), code, False, c))
                for a, o, c in zip(xb, yb, caps)]
        cb = [np.empty(len(r), dtype=np.int32) for r in S.rows]
        batches = bs

        def call(lens):
            for p in range(len(bs)):
                torch.index_select(x, 0, idx[p], out=xb[p])
                lp = np.ascontiguousarray(lens[S.rows[p]])
                if fn(bs[p]._h, C.byref(bufs[p][0]), lp.ctypes.data, C.byref(bufs[p][1]), caps[p], cb[p].ctypes.data) < 0:
                    raise pkg.R8bGpuError(pkg._err())
                y[:, :caps[p]].index_copy_(0, idx[p], yb[p])
                counts[S.rows[p]] = cb[p]

    for i in range(warmup):
        call(lens_c[i])
    torch.cuda.synchronize()
    l0 = sum(b.kernel_launches for b in batches)
    t0 = time.perf_counter()
    n_in = 0
    for lens in lens_c[warmup:]:
        call(lens)
        n_in += int(lens.sum())
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    steps = len(lens_c) - warmup
    return {"case": case, "format": fmt, "form": "host" if host else "device", "channels": n_ch,
            "block_len": "%d..%d" % (int(np.min(lens_seq)), int(np.max(lens_seq))),
            "in_gsamples_per_s": n_in / dt / 1e9, "ms_per_call": 1e3 * dt / steps,
            "launches_per_call": (sum(b.kernel_launches for b in batches) - l0) / steps}


def profile_share(pkg, torch, S, lens_seq):
    """Share of the kernel time of mixed device fp64 calls spent in the mapped conversions (k_cvt_*)."""
    from torch.profiler import ProfilerActivity, profile
    L = pkg.lib()
    b = pkg.Batch.mixed(S.plans, S.plan_of, 0)
    b.set_stream(torch.cuda.current_stream().cuda_stream)
    cap = b.max_out_len
    x = torch.rand((S.n_ch, MAX_IN), dtype=torch.float64, device="cuda:0") * 2 - 1
    y = torch.empty((S.n_ch, cap), dtype=torch.float64, device="cuda:0")
    counts = np.empty(S.n_ch, dtype=np.int32)
    lens_c = [np.ascontiguousarray(v, dtype=np.int32) for v in lens_seq]

    def call(lens):
        if L.r8bgpu_batch_process_ragged(b._h, x.data_ptr(), MAX_IN, lens.ctypes.data, y.data_ptr(), cap, cap,
                                         counts.ctypes.data) < 0:
            raise pkg.R8bGpuError(pkg._err())
    for lens in lens_c[:2]:
        call(lens)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for lens in lens_c[2:]:
            call(lens)
        torch.cuda.synchronize()
    tot = cvt = 0.0
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = e.cuda_time_total
        if "memcpy" in e.key.lower() or "memset" in e.key.lower():
            continue
        tot += t
        if "k_cvt_" in e.key:
            cvt += t
    return {"case": "mixed", "profile": "f64 device", "calls": len(lens_c) - 2, "kernel_ms": tot / 1e3,
            "mapped_conversion_ms": cvt / 1e3, "mapped_conversion_share": cvt / tot if tot else 0.0}


def verify(pkg, S, lens, n_sample=12):
    """A fresh mixed batch's first call against the reference on sampled channels (counts equal, parity bar)."""
    import oracle_util as ou
    if not ou.have_ref("e0"):
        return {"verify": "skipped: oracle/_ref not built"}
    ref = ou.RefOracle("e0")
    b = pkg.Batch.mixed(S.plans, S.plan_of, 0)
    x = ou.white_noise(S.n_ch, MAX_IN, 3)
    ys = b.process_ragged([x[c, :lens[c]] for c in range(S.n_ch)])
    worst = 0.0
    chans = np.random.default_rng(5).choice(S.n_ch, n_sample, replace=False)
    for c in chans:
        r = ref.Resampler(RATES[S.plan_of[c]], DST, MAX_IN, 2.0, pkg.ATTEN_24).process(x[c, :lens[c]])
        assert len(r) == len(ys[c]), (c, len(r), len(ys[c]))
        if np.any(r):
            m, rms = ou.parity_metrics(ys[c], r)
            assert m <= 32 * ou.EPS and rms <= 4 * ou.EPS, (c, m / ou.EPS, rms / ou.EPS)
            worst = max(worst, m / ou.EPS)
    return {"verify": "ok", "channels_checked": len(chans), "worst_max_err_eps": worst}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--channels", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--min-len", type=int, default=32768)
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--formats", default="f64,s16")
    ap.add_argument("--cases", default="mixed,buckets")
    ap.add_argument("--label", default=None)
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    import torch
    from __graft_entry__ import load_package
    pkg = load_package()
    if not torch.cuda.is_available():
        raise SystemExit("mixed_bench: no CUDA device")
    S = Setup(pkg, torch, args.channels, args.seed)
    rng = np.random.default_rng(args.seed)
    lens_seq = rng.integers(args.min_len, MAX_IN + 1, size=(args.warmup + args.steps, args.channels))
    gpu = torch.cuda.get_device_name(0)
    q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    power = q.stdout.strip() if q.returncode == 0 else "unknown"
    tag = {"gpu": gpu, "power_limit": power}
    if args.label:
        tag["label"] = args.label
    print(json.dumps(dict(verify(pkg, S, lens_seq[0]), **tag)), flush=True)
    for fmt in args.formats.split(","):
        for host in (False, True):
            for case in args.cases.split(","):
                r = run(pkg, torch, S, case, fmt, host, lens_seq, args.warmup)
                print(json.dumps(dict(r, **tag)), flush=True)
    if args.profile:
        print(json.dumps(dict(profile_share(pkg, torch, S, lens_seq[:8]), **tag)), flush=True)


if __name__ == "__main__":
    main()
