#!/usr/bin/env python3
"""TEST INFRASTRUCTURE: random-configuration campaign for the emulated library (tests/emu).

    python tests/emu/fuzz.py <seed> <seconds>

Random frame size (1..700 px), strategy subset, Gaborish/EPF setting, coefficient type, output format,
transfer function, stage chain (incl. odd ones -> tile kernel) and hand-off (dense / sparse / shuffled /
streamed / band by band); every frame is compared bit for bit with the oracle.  End of round 1: 872
frames over four seeds, no mismatch.  Round 2 adds: EPF engaged on a random subset of the blocks (sharpness 0 / 7,
quantiser 1: the strip kernel's block permutation), upsampling 2/4/8 with ragged output sizes, noise.  Half of the
frames carry a random legal non-default frame header (jxl_workload.header_params: Gaborish weights, EPF LUT and
scales, CfL base, colour factor, quantisation biases, qm scales, opsin matrix and biases, intensity target)."""
import sys, time, ctypes as C
from pathlib import Path
sys.path.insert(0, str(Path(__file__).resolve().parents[2]))
import numpy as np
import jxl_workload as wl
from libjxl_b200 import abi, pipeline, sharding
from tests.emu import build_emu
from oracle import cpu
pipeline._lib = pipeline.bind(C.CDLL(str(build_emu.build())))
pipe = pipeline.TransformPipeline(device=0, num_host_threads=2)
WTS = np.load(Path(__file__).resolve().parents[1] / "golden" / "upsampling_weights.npz")
rng = np.random.default_rng(int(sys.argv[1]) if len(sys.argv)>1 else 0)
t_end = time.time() + float(sys.argv[2]) if len(sys.argv)>2 else time.time()+300
n=0; bad=0
def same(a,b):
    if a.dtype==np.float16: a,b=a.view(np.uint16),b.view(np.uint16)
    return a.shape==b.shape and np.array_equal(a,b)
while time.time() < t_end:
    w = int(rng.integers(1, 420)); h = int(rng.integers(1, 420))
    if rng.random()<0.15: w = int(rng.integers(500, 700))
    gab = int(rng.integers(0,2)); epf = int(rng.integers(0,4)); ac = int(rng.integers(0,2))
    fmt = int(rng.integers(0,6)); srgb = abi.STAGE_SRGB if rng.random()<0.5 else 0
    strategies = "all" if rng.random()<0.7 else ",".join(str(int(s)) for s in rng.choice(27, int(rng.integers(1,6)), replace=False))
    try:
        desc, coeffs = wl.synthetic_frame(w, h, seed=int(rng.integers(1<<30)), gab=gab, epf_iters=epf, ac_type=ac, strategies=strategies)
    except Exception as e:
        desc, coeffs = wl.synthetic_frame(w, h, seed=int(rng.integers(1<<30)), gab=gab, epf_iters=epf, ac_type=ac)
    desc.out_format, desc.stage_mask = fmt, srgb
    hdr = int(rng.integers(1 << 30)) if rng.random() < 0.5 else None
    if hdr is not None:
        wl.apply_header(desc, wl.header_params(hdr))
    post = False
    if epf and rng.random() < 0.5:   # EPF really engaged on part of the blocks
        desc.raw_quant = np.where(desc.raw_quant > 0, 1, 0).astype(np.int32)
        desc.epf_sharpness = np.where(rng.random(desc.epf_sharpness.shape) < rng.random(), 7, 0).astype(np.uint8)
        coeffs = np.clip(coeffs, -2, 2)
    if rng.random() < 0.25 and w * h < 40000:   # upsampling and / or noise (whole-frame features)
        post = True
        if rng.random() < 0.7:
            nn = int(rng.choice([2, 4, 8]))
            desc.upsampling, desc.upsampling_weights = nn, WTS[f"weights{nn}"]
            desc.xsize_upsampled = nn * w - int(rng.integers(0, nn)); desc.ysize_upsampled = nn * h - int(rng.integers(0, nn))
        if desc.upsampling == 1 or rng.random() < 0.5:
            desc.noise, desc.noise_lut = 1, tuple(float(x) for x in rng.random(8) * 0.02)
            desc.visible_frame_index, desc.nonvisible_frame_index = int(rng.integers(0, 5)), int(rng.integers(0, 3))
    if not post and rng.random()<0.2:  # explicit odd chain -> tile kernel
        desc.stage_mask = abi.STAGE_EXPLICIT | int(rng.integers(0,32)) | srgb
        if (desc.stage_mask & 14) and epf==0: desc.stage_mask &= ~14
    want = cpu.render_frame(desc, coeffs, rcp_mode=0)
    mode = rng.integers(0,3) if post else rng.integers(0,4)
    cfg = dict(w=w,h=h,gab=gab,epf=epf,ac=ac,fmt=fmt,mask=hex(desc.stage_mask),mode=int(mode),ups=desc.upsampling,noise=desc.noise,hdr=hdr)
    try:
        if mode==0: got = pipe.decode_frame(desc, coeffs)
        elif mode==1: got = pipe.decode_frame(desc, coeffs, sparse=True, order=rng.permutation(desc.num_groups).tolist(), stream_output=True)
        elif mode==2: got = pipe.decode_frame(desc, coeffs, order=rng.permutation(desc.num_groups).tolist(), stream_output=bool(rng.integers(0,2)))
        else:
            world = int(rng.integers(1, 4)); rows=[]
            for (y0, ny) in sharding.band_partition(desc.ysize_groups, world):
                if ny==0: continue
                desc.band_y0_groups, desc.band_ny_groups = y0, ny
                pipe.set_device_coefficients(None); pipe.frame_begin(desc)
                for g in sharding.groups_needed(desc, y0, ny): pipe.submit_group(g, [coeffs[c,g] for c in range(3)])
                rows.append(pipe.frame_finish())
            desc.band_y0_groups = desc.band_ny_groups = 0
            got = np.concatenate(rows, axis=1 if fmt==abi.OUT_PLANAR_F32 else 0)
        ok = same(got, want)
    except Exception as e:
        ok = False; print("EXC", cfg, repr(e), flush=True)
    n+=1
    if not ok:
        bad+=1; print("MISMATCH", cfg, flush=True)
print(f"seed {sys.argv[1] if len(sys.argv)>1 else 0}: {n} frames, {bad} bad", flush=True)
