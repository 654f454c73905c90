"""A/B of the matrix-path tilings of one separable pass: the 8192^2 RGBA BlurImage(0,4) row and column passes (33 taps,
conv_mma.cu) with mma_wide 0 (DMMA.8x8x4 tiles) and 1 (DMMA.16x8x16 tiles), alternating in one process.

Prints the median, min and max of >= 20 CUDA-event timed repetitions per pass and arm, the share of 3.35 TB/s at 32 B/px,
the number of samples in which the two arms differ (and by how many ULP at most) on the full image, and both arms against
the oracle on a 1031 x 517 crop.  Writes the JSON record to --out when given.

    python tools/conv_ab.py [--reps 30] [--rounds 3] [--option mma_strip=1024] [--out conv_ab.json]
"""
from __future__ import annotations

import argparse
import json
import statistics
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))

import imagemagick_b200 as im  # noqa: E402
import util  # noqa: E402

SIZE, SIGMA = 8192, 4.0
HBM = 3.35e12


def ulp_stats(a: torch.Tensor, b: torch.Tensor):
    ia, ib = a.view(torch.int32).to(torch.int64), b.view(torch.int32).to(torch.int64)
    ia = torch.where(ia < 0, -(ia & 0x7FFFFFFF), ia)
    ib = torch.where(ib < 0, -(ib & 0x7FFFFFFF), ib)
    d = (ia - ib).abs()
    return int((d != 0).sum()), int(d.max())


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=3, help="alternations of the two arms")
    ap.add_argument("--option", action="append", default=[], metavar="NAME=VALUE",
                    help="a run-time option set for both arms, e.g. mma_strip=1024")
    ap.add_argument("--out", type=Path)
    args = ap.parse_args()
    options = {k: int(v) for k, v in (o.split("=", 1) for o in args.option)}
    assert torch.cuda.is_available(), "conv_ab.py times kernels on cuda:0"
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    g = torch.Generator(device="cuda").manual_seed(7)
    x = torch.rand((SIZE, SIZE, 4), device="cuda", generator=g) * 65535.0
    x[..., 3] = torch.where(x[..., 3] < 6553.5, torch.zeros_like(x[..., 3]), x[..., 3])       # some transparent pixels
    src = im.Image(x)
    kernels = {"row": im.AcquireKernelInfo(f"blur:0x{SIGMA:g}"), "column": im.AcquireKernelInfo(f"blur:0x{SIGMA:g}+90")}

    times = {(p, w): [] for p in kernels for w in (0, 1)}
    outs = {}
    for _ in range(args.rounds):
        for wide in (0, 1):
            for name, v in options.items():
                util.set_option(name, v)
            util.set_option("mma_wide", wide)
            for p, k in kernels.items():
                n0 = util.get_option("conv_mma_wide_launches")
                out = im.ConvolveImage(src, k)                                   # warm-up, and the result compared below
                assert (util.get_option("conv_mma_wide_launches") - n0) == wide, (p, wide)
                outs[(p, wide)] = out.pixels
                torch.cuda.synchronize()
                for _ in range(args.reps // args.rounds + 1):
                    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    a.record()
                    im.ConvolveImage(src, k)
                    b.record()
                    torch.cuda.synchronize()
                    times[(p, wide)].append(a.elapsed_time(b))

    rec = {"gpu": gpu, "size": SIZE, "sigma": SIGMA, "options": options, "passes": {}}
    for p in kernels:
        for wide in (0, 1):
            ts = times[(p, wide)]
            med = statistics.median(ts)
            rec["passes"][f"{p}_wide{wide}"] = {"n": len(ts), "median_ms": med, "min_ms": min(ts), "max_ms": max(ts),
                                               "hbm_share_32Bpx": 32.0 * SIZE * SIZE / (med * 1e-3) / HBM}
        n, mx = ulp_stats(outs[(p, 0)], outs[(p, 1)])
        rec["passes"][f"{p}_bits"] = {"differing_samples": n, "max_ulp": mx, "samples": SIZE * SIZE * 4}

    # both arms against the oracle on a crop (whole-image passes of a 1031 x 517 image: ragged strips on both axes)
    crop = x[:517, :1031].contiguous()
    crop_np = crop.cpu().numpy()
    for p, k in kernels.items():
        (values, ox, oy), = k.arrays()
        want = util.orc_morphology(crop_np, im.ConvolveMorphology, 1, [util.orc_kernel_from_array(values, ox, oy)])
        for wide in (0, 1):
            util.set_option("mma_wide", wide)
            got = im.ConvolveImage(im.Image(crop), k).pixels.cpu().numpy()
            d = util.ulp_distance(got, want)
            rec["passes"][f"{p}_wide{wide}_oracle"] = {"max_ulp": int(d.max()), "frac_exact": float((d == 0).mean())}
    util.reset_options()

    print(json.dumps(rec, indent=1))
    if args.out:
        args.out.parent.mkdir(parents=True, exist_ok=True)
        args.out.write_text(json.dumps(rec, indent=1))


if __name__ == "__main__":
    main()
