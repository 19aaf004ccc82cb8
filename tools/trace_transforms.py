#!/usr/bin/env python3
"""Where the inverse transforms run inside a render: a torch.profiler trace (CUDA activities) of a few
`render_device` steps of one bench.py frame (default `8k-d1`, f32) in normal mode, i.e. with the mid and large
transforms on their side streams beside the 8x8 kernel.  For every step it prints each kernel's start and end
(µs from the step's plan kernel) and its stream; then, per build, the mean span of the 8x8 kernel in the trace
against its time alone in the profiling pass (`kernel_times_ms()["idct8"]`, where the kernels run one after the
other on one stream).

    python tools/trace_transforms.py [--workload 8k-d1] [--steps 5] [--rounds 2] [--out DIR] [--compare DIR]

--compare DIR traces DIR's build (DIR/libjxl_b200/libjxl_b200.so) in the same process, alternating with this tree's
build round by round.  The chrome traces go to --out (default: a new temporary directory), one per build and round."""
import argparse
import ctypes as C
import json
import sys
import tempfile
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

import numpy as np  # noqa: E402

import jxl_workload as wl  # noqa: E402
from bench import WORKLOADS, ClockSampler  # noqa: E402
from libjxl_b200 import abi, pipeline  # noqa: E402
from tools.measure_strip_filter import card  # noqa: E402

SHORT = (("plan_kernel", "plan"), ("idct8_tma_kernel", "idct8"), ("idct8_kernel", "idct8"),
         ("idct_mid_kernel", "mid"), ("idct_large_kernel<true, 0>", "large0"), ("idct_large_kernel<false, 0>", "large0"),
         ("idct_large_kernel<true, 1>", "large1"), ("idct_large_kernel<false, 1>", "large1"),
         ("filter_strip_kernel", "filter"), ("filter_kernel", "filter"))


def short_name(name: str) -> str:
    for k, v in SHORT:
        if k in name:
            return v
    return name.split("(")[0][:40]


def trace_steps(L, desc, ptrs, out, steps: int, warmup: int, path: Path) -> list:
    """Kernels of `steps` traced render_device calls with library `L`: one list of
    (name, stream, start_us, end_us) per step, times relative to the step's plan kernel."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    saved = pipeline._lib
    pipeline._lib = L
    try:
        pipe = pipeline.TransformPipeline(device=0)
        try:
            pipe.set_device_coefficients(ptrs)
            pipe.frame_begin(desc)
            for _ in range(warmup):
                pipe.render_device(out.data_ptr(), desc.out_row_bytes)
            pipe.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(steps):
                    pipe.render_device(out.data_ptr(), desc.out_row_bytes)
                pipe.synchronize()
                torch.cuda.synchronize()
            prof.export_chrome_trace(str(path))
            pipe.set_profiling(True)
            alone = []
            for _ in range(20):
                pipe.render_device(out.data_ptr(), desc.out_row_bytes)
                alone.append(pipe.kernel_times_ms())
            pipe.set_profiling(False)
            pipe.set_device_coefficients(None)
        finally:
            pipe.close()
    finally:
        pipeline._lib = saved
    ev = [e for e in json.loads(path.read_text())["traceEvents"] if e.get("cat") == "kernel"]
    ev.sort(key=lambda e: e["ts"])
    res, cur = [], None
    for e in ev:
        n = short_name(e["name"])
        if n == "plan":
            cur = []
            res.append(cur)
        if cur is None:
            continue
        cur.append((n, e["args"].get("stream"), float(e["ts"]), float(e["ts"]) + float(e["dur"])))
    for st in res:
        t0 = st[0][2]
        st[:] = [(n, s, a - t0, b - t0) for n, s, a, b in st]
    return res, {k: float(np.mean([a[k] for a in alone])) for k in alone[0]}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--workload", default="8k-d1", choices=[k for k, v in WORKLOADS.items() if v[6] != "noise"])
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--out", default=None, help="directory for the chrome traces (default: a new temporary one)")
    ap.add_argument("--compare", metavar="DIR", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("no CUDA device: this tool traces the GPU and has no CPU path")
    outdir = Path(args.out) if args.out else Path(tempfile.mkdtemp(prefix="trace_transforms_"))
    outdir.mkdir(parents=True, exist_ok=True)

    w, h, dist, effort, gab, epf, kind = WORKLOADS[args.workload]
    if kind == "synthetic-all-strategies":   # as bench.py makes it
        desc, coeffs = wl.synthetic_frame(w, h, seed=1234, gab=gab, epf_iters=epf)
    else:
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
    print(f"traces: {outdir}")
    print(f"card: {info}  workload {args.workload} ({desc.xsize}x{desc.ysize}), {args.steps} traced steps "
          f"after {args.warmup} warm-up, {args.rounds} rounds", flush=True)

    summary = {n: {"idct8_span": [], "idct8_alone": [], "step_span": [], "transforms_span": []} for n in libs}
    sampler = ClockSampler(0)
    sampler.start()
    for rnd in range(args.rounds):
        for li, (name, L) in enumerate(libs.items()):
            steps, alone = trace_steps(L, desc, ptrs, out, args.steps, args.warmup,
                                       outdir / f"{args.workload}_lib{li}_round{rnd}.pt.trace.json")
            print(f"\nround {rnd} {name}: profiling pass (serial, ms) " +
                  "  ".join(f"{k} {v:.4f}" for k, v in alone.items()))
            for si, st in enumerate(steps):
                print(f"  step {si}: " + "  ".join(f"{n}[s{s}] {a:7.1f}..{b:7.1f}" for n, s, a, b in st))
                by = {n: (a, b) for n, s, a, b in st}
                if "idct8" not in by or "filter" not in by:
                    continue
                summary[name]["idct8_span"].append(by["idct8"][1] - by["idct8"][0])
                summary[name]["step_span"].append(by["filter"][1])
                summary[name]["transforms_span"].append(by["filter"][0] - by["plan"][1])
            summary[name]["idct8_alone"].append(alone["idct8"] * 1000.0)
    clocks = sampler.stop()
    print(f"\nSM clock under load {clocks.get('sm_mhz')} MHz (max {clocks.get('sm_max_mhz')}), "
          f"throttle reasons {clocks.get('reasons')}")
    print("\nmeans over traced steps, µs: 8x8 span in the trace | 8x8 alone (profiling pass) | "
          "plan end -> filter start | plan start -> filter end")
    for n, s in summary.items():
        print(f"  {n:>10}: {np.mean(s['idct8_span']):7.1f} | {np.mean(s['idct8_alone']):7.1f} | "
              f"{np.mean(s['transforms_span']):7.1f} | {np.mean(s['step_span']):7.1f}")
    print(json.dumps({"card": info, "clocks": clocks, "workload": args.workload,
                      "summary_us": {n: {k: float(np.mean(v)) for k, v in s.items()} for n, s in summary.items()}}))


if __name__ == "__main__":
    main()
