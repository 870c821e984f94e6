"""Time the 16-bit moment kernels against the float32 tf32x3b kernel and today's float64-copy route of 16-bit data.

One process, CUDA events, warm-up, variants alternated within each repetition, medians reported.  Per shape:
  * ops.moments on float32 views (tf32x3b), on bf16 views and on fp16 views (the 16-bit wgmma kernel);
  * bf16 views by the float64-copy route: v.double() then the DMMA kernel, the conversion included;
  * rCCA(latent_dimensions=64, c=0.1).fit on bf16 CUDA views against the same fit on their float64 copy.
Achieved TFLOP/s counts n * D * (D + 1) (the upper triangle and the column sums as the kernels do it: 2 flop per
multiply-add over the D (D + 1) / 2 entries), and the share of peak is the larger of that work at the data sheet's dense
BF16 rate and the bytes of the views at its HBM3 bandwidth, over the kernel time; the line names which bound applies.
The moments of the variants are compared at the timed sizes against the bound of tests/test_moments_half_gpu.py.

Usage: python tools/bench_half_moments.py [--reps 7]
"""
from __future__ import annotations

import argparse
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from cca_zoo_b200 import ops  # noqa: E402
from cca_zoo_b200.linear import rCCA  # noqa: E402

PEAK_BF16 = 989e12     # H100 SXM data sheet, dense BF16 / FP16, 700 W
PEAK_HBM = 3.35e12     # bytes / s
SHAPES = [(100_000, [1024, 1024]), (200_000, [4096, 4096])]
BOUND = 256 * 2.0 ** -23     # normalised moment error bound of the 16-bit kernel (see the tests)


def _card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        q = "unknown"
    return name, q


def _time(fn, reps_inner=3):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps_inner):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / reps_inner


def _normalised_err(M, ref, Dp):
    M, ref = M[:Dp * Dp].reshape(Dp, Dp), ref[:Dp * Dp].reshape(Dp, Dp)
    d = torch.diagonal(ref).clamp_min(1e-300)
    return ((M - ref).abs().triu() / torch.sqrt(d[:, None] * d[None, :])).max().item()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_half_moments needs a CUDA device")
    name, q = _card()
    print(f"GPU: {name}; power.limit, clocks.max.sm: {q}")
    for n, dims in SHAPES:
        D = sum(dims)
        g = torch.Generator(device="cuda").manual_seed(0)
        v32 = [torch.randn(n, d, generator=g, device="cuda") for d in dims]
        vb = [x.bfloat16() for x in v32]
        vh = [x.half() for x in v32]
        vb32 = [x.float() for x in vb]          # the bf16 values as float32: same data for tf32x3b
        variants = {
            "f32 tf32x3b": lambda: ops.moments(vb32, precision="tf32x3b"),
            "bf16 wgmma": lambda: ops.moments(vb, precision="tf32x3b"),
            "fp16 wgmma": lambda: ops.moments(vh, precision="tf32x3b"),
            "bf16 via f64": lambda: ops.moments([x.double() for x in vb], precision="exact"),
        }
        # results at the timed size
        ref_b = ops.moments([x.double() for x in vb], precision="exact")
        ref_h = ops.moments([x.double() for x in vh], precision="exact")
        Dp = int(round((-1 + (1 + 4 * ref_b.numel()) ** 0.5) / 2))
        errs = {"f32 tf32x3b": _normalised_err(variants["f32 tf32x3b"](), ref_b, Dp),
                "bf16 wgmma": _normalised_err(variants["bf16 wgmma"](), ref_b, Dp),
                "fp16 wgmma": _normalised_err(variants["fp16 wgmma"](), ref_h, Dp)}
        del ref_b, ref_h
        for k in variants:                       # warm-up
            variants[k]()
        torch.cuda.synchronize()
        times = {k: [] for k in variants}
        for _ in range(args.reps):
            for k, fn in variants.items():       # alternated
                times[k].append(_time(fn, 1 if k == "bf16 via f64" else 3))
        flop = n * D * (D + 1)
        print(f"\nshape n = {n}, dims = {dims}: {flop:.3e} flop")
        med = {k: sorted(t)[len(t) // 2] for k, t in times.items()}
        for k, ms in med.items():
            byts = n * D * (4 if k == "f32 tf32x3b" else 2)
            t_flop, t_mem = flop / PEAK_BF16, byts / PEAK_HBM
            bound = "BF16 tensor" if t_flop >= t_mem else "HBM"
            share = max(t_flop, t_mem) / (ms * 1e-3)
            err = f", max normalised error {errs[k]:.2e} (bound {BOUND:.2e})" if k in errs else ""
            print(f"  {k:14s} {ms:8.3f} ms  {flop / (ms * 1e-3) / 1e12:7.1f} TFLOP/s  {100 * share:5.1f} % of the "
                  f"data-sheet {bound} bound{err}")
        for k in ("bf16 wgmma", "fp16 wgmma"):
            print(f"  speed-up of {k} over f32 tf32x3b: {med['f32 tf32x3b'] / med[k]:.2f}x")
        for k, e in errs.items():
            if k != "f32 tf32x3b" and e > BOUND:
                raise SystemExit(f"{k}: moments differ from float64 by {e:.2e} > {BOUND:.2e}")
        del vh, v32, vb32
        if D <= 2048:
            # end to end: rCCA on bf16 CUDA views vs on their float64 copy (the copy included in its time)
            est = rCCA(latent_dimensions=64, c=0.1)
            fits = {"rCCA.fit bf16 views": lambda: est.fit(vb),
                    "rCCA.fit f64 copy": lambda: est.fit([x.double() for x in vb])}
            for fn in fits.values():
                fn()
            ft = {k: [] for k in fits}
            for _ in range(args.reps):
                for k, fn in fits.items():
                    torch.cuda.synchronize()
                    ft[k].append(_time(fn, 1))
            for k, t in ft.items():
                print(f"  {k:20s} {sorted(t)[len(t) // 2]:8.3f} ms (median of {len(t)})")
        del vb
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
