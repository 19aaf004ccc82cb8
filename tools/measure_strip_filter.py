#!/usr/bin/env python3
"""Decomposes the strip filter's time by stage chain: render_device of one bench.py frame (default `8k-d1`, the same
cached reference-encoded frame bench.py uses) with each explicit chain, `kernel_ms["filter"]` averaged over many
profiled launches after a warm-up.  The differences between chains give the cost of each stage, e.g.
filter(17) - filter(16) is the whole cost of Gaborish.

    python tools/measure_strip_filter.py [--workload 8k-d1] [--launches 30] [--rounds 3] [--compare DIR]

--compare DIR times DIR's build (DIR/libjxl_b200/libjxl_b200.so, e.g. a checkout of another commit after its build())
in the same process, alternating with this tree's build round by round.  Prints the card name, power limit and the
SM clock sampled while the timed launches ran."""
import argparse
import ctypes as C
import json
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

import numpy as np  # noqa: E402

import jxl_workload as wl  # noqa: E402
from bench import WORKLOADS, ClockSampler  # noqa: E402
from libjxl_b200 import abi, pipeline  # noqa: E402

# 16 = XYB only, 17 = + Gaborish, 20 = EPF1 + XYB, 21 = Gaborish + EPF1 + XYB (8k-d1's own chain),
# 29 = Gaborish + EPF1 + EPF2 + XYB, 31 = all three EPF passes
CHAINS = (16, 17, 20, 21, 29, 31)


def card() -> dict:
    q = "name,power.limit,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", "--id=0", f"--query-gpu={q}", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        name, plim, smax = [x.strip() for x in r.stdout.strip().split(",")]
        return {"name": name, "power_limit": plim, "sm_max_clock": smax}
    except Exception as e:  # noqa: BLE001
        return {"error": repr(e)}


def time_chains(L, desc, ptrs, out, launches: int, warmup: int) -> dict:
    """Mean filter-kernel time (ms) per chain with library `L`."""
    saved = pipeline._lib
    pipeline._lib = L
    res = {}
    try:
        pipe = pipeline.TransformPipeline(device=0)
        try:
            pipe.set_device_coefficients(ptrs)
            for chain in CHAINS:
                desc.stage_mask = abi.STAGE_EXPLICIT | chain
                pipe.frame_begin(desc)
                for _ in range(warmup):
                    pipe.render_device(out.data_ptr(), desc.out_row_bytes)
                pipe.synchronize()
                pipe.set_profiling(True)
                t = []
                for _ in range(launches):
                    pipe.render_device(out.data_ptr(), desc.out_row_bytes)
                    t.append(pipe.kernel_times_ms()["filter"])
                pipe.set_profiling(False)
                res[chain] = float(np.mean(t))
            pipe.set_device_coefficients(None)
        finally:
            pipe.close()
    finally:
        pipeline._lib = saved
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--workload", default="8k-d1", choices=[k for k, v in WORKLOADS.items() if v[6] == "photo"])
    ap.add_argument("--launches", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--compare", metavar="DIR", default=None)
    args = ap.parse_args()
    if args.launches < 20:
        ap.error("--launches must be at least 20")
    import torch
    if not torch.cuda.is_available():
        sys.exit("no CUDA device: this tool measures the GPU and has no CPU path")

    w, h, dist, effort, gab, epf, kind = WORKLOADS[args.workload]
    fr = wl.reference_frame(w, h, dist, effort, gab, epf, seed=1234, kind=kind, cache=True)
    desc, coeffs = fr["desc"], fr["coeffs"]
    desc.out_format = abi.OUT_RGB_F32
    dev = torch.from_numpy(coeffs).cuda()
    ptrs = [dev[c].data_ptr() for c in range(3)]
    out = torch.empty((desc.ysize, desc.xsize, 3), dtype=torch.float32, device="cuda")

    libs = {"this tree": pipeline.lib()}
    if args.compare:
        so = Path(args.compare).resolve() / "libjxl_b200" / "libjxl_b200.so"
        libs["compare"] = pipeline.bind(C.CDLL(str(so)))
    info = card()
    print(f"card: {info}  workload {args.workload} ({w}x{h}, gab={desc.gab}, epf={desc.epf_iters}), "
          f"{args.launches} profiled launches per chain after {args.warmup} warm-up", flush=True)

    times = {k: {c: [] for c in CHAINS} for k in libs}
    sampler = ClockSampler(0)
    sampler.start()
    for rnd in range(args.rounds):
        for name, L in libs.items():
            r = time_chains(L, desc, ptrs, out, args.launches, args.warmup)
            for c, v in r.items():
                times[name][c].append(v)
            print(f"round {rnd} {name}: " + "  ".join(f"{c}: {v:.4f}" for c, v in r.items()), flush=True)
    clocks = sampler.stop()
    print(f"SM clock under load {clocks.get('sm_mhz')} MHz (max {clocks.get('sm_max_mhz')}), "
          f"throttle reasons {clocks.get('reasons')}")

    print("\nfilter kernel ms, mean over rounds (min..max of the round means)")
    print("chain  " + "  ".join(f"{n:>24}" for n in libs))
    for c in CHAINS:
        print(f"{c:5d}  " + "  ".join(f"{np.mean(times[n][c]):8.4f} ({min(times[n][c]):.4f}..{max(times[n][c]):.4f})"
                                      for n in libs))
    for n in libs:
        m = {c: float(np.mean(v)) for c, v in times[n].items()}
        print(f"{n}: Gaborish = filter(17) - filter(16) = {m[17] - m[16]:.4f} ms; "
              f"in chain 21: filter(21) - filter(20) = {m[21] - m[20]:.4f} ms")
    print(json.dumps({"card": info, "clocks": clocks, "workload": args.workload,
                      "filter_ms": {n: {str(c): v for c, v in t.items()} for n, t in times.items()}}))


if __name__ == "__main__":
    main()
