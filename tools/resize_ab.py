"""A/B of ResizeImage's two paths for equal 2x reductions of RGBA images: the two streaming passes (vertical into a
temporary, then horizontal) against the fused vertical + horizontal kernel.  Both arms run in one process, alternating,
timed with CUDA events on device-resident images; every pair of results is compared bit for bit.

usage: python tools/resize_ab.py [--reps R] [--rounds K] [--sizes 1024,2048,...] [--json PATH]

Each row reports the median time per call, the effective rate over the path's own HBM byte count (two passes:
16 + 8 B per source pixel for the vertical pass, 8 + 4 for the horizontal one = 36 B/px; fused: 16 + 4 = 20 B/px) and
its share of the H100 SXM's 3.35 TB/s, and which path the automatic selection takes at that size."""
import argparse
import ctypes as C
import json
import subprocess
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import torch  # noqa: E402

import imagemagick_b200 as im  # noqa: E402
from imagemagick_b200 import _lib  # noqa: E402

HBM_PEAK = 3.35e12            # H100 SXM data sheet, bytes/s
BYTES_TWO_PASS, BYTES_FUSED = 36, 20


def option(name):
    v = C.c_int(0)
    _lib.check(_lib.load().mb200_get_option(name.encode(), C.byref(v)))
    return v.value


def set_option(name, value):
    _lib.check(_lib.load().mb200_set_option(name.encode(), int(value)))


def card():
    q = "name,power.limit,clocks.max.sm,memory.total"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
    except (OSError, subprocess.SubprocessError):
        out = []
    return out[torch.cuda.current_device()] if out else torch.cuda.get_device_name()


ARMS = {"two_pass": {"resize_fused": 0, "no_resize_fused": 1}, "fused": {"resize_fused": 1, "no_resize_fused": 0},
        "auto": {"resize_fused": 0, "no_resize_fused": 0}}


def run(arm, fn):
    for k, v in ARMS[arm].items():
        set_option(k, v)
    return fn()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--sizes", default="1024,2048,4096,8192,16384")
    ap.add_argument("--json", default="")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "resize_ab.py times the GPU kernels and needs a CUDA device"
    print("card:", card(), "| L2", torch.cuda.get_device_properties(0).L2_cache_size >> 20, "MiB", flush=True)
    rows = []
    g = torch.Generator(device="cuda").manual_seed(5)
    for filt_name, filt in (("Lanczos", im.LanczosFilter), ("Mitchell", im.MitchellFilter)):
        for n in (int(s) for s in args.sizes.split(",")):
            src = im.Image(torch.rand(n, n, 4, device="cuda", generator=g) * 65535)
            call = lambda: im.ResizeImage(src, n // 2, n // 2, filt)   # noqa: E731
            outs, times = {}, {arm: [] for arm in ARMS}
            for arm in ARMS:                                   # warm-up: tables, pools, modules
                outs[arm] = run(arm, call).pixels.clone()
            before = option("resize_fused_launches")
            run("auto", call)
            auto_fused = option("resize_fused_launches") > before
            torch.cuda.synchronize()
            for _ in range(args.rounds):
                for arm in ("two_pass", "fused"):
                    run(arm, lambda: None)
                    for _ in range(args.reps):
                        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        a.record(); call(); b.record()
                        b.synchronize()
                        times[arm].append(a.elapsed_time(b))
            identical = torch.equal(outs["two_pass"], outs["fused"]) and torch.equal(outs["auto"], outs["fused"])
            row = {"filter": filt_name, "size": n, "identical": identical, "auto": "fused" if auto_fused else "two_pass"}
            for arm, bpp in (("two_pass", BYTES_TWO_PASS), ("fused", BYTES_FUSED)):
                t = sorted(times[arm])
                ms = t[len(t) // 2]
                row[arm + "_ms"] = round(ms, 4)
                row[arm + "_min_ms"] = round(t[0], 4)
                row[arm + "_hbm_frac"] = round(n * n * bpp / (ms * 1e-3) / HBM_PEAK, 3)
            row["speedup"] = round(row["two_pass_ms"] / row["fused_ms"], 3)
            rows.append(row)
            print(f"{filt_name:8s} {n:5d}^2 -> {n // 2:5d}^2  two-pass {row['two_pass_ms']:8.3f} ms "
                  f"({row['two_pass_hbm_frac'] * 100:5.1f}% of 3.35 TB/s at 36 B/px)  fused {row['fused_ms']:8.3f} ms "
                  f"({row['fused_hbm_frac'] * 100:5.1f}% at 20 B/px)  x{row['speedup']:.2f}  auto={row['auto']:8s} "
                  f"bits {'identical' if identical else 'DIFFER'}", flush=True)
            del src, outs
            torch.cuda.empty_cache()
    for k in ("resize_fused", "no_resize_fused"):
        set_option(k, 0)
    if args.json:
        Path(args.json).parent.mkdir(parents=True, exist_ok=True)
        Path(args.json).write_text(json.dumps({"card": card(), "rows": rows}, indent=1))
    if not all(r["identical"] for r in rows):
        sys.exit("fused and two-pass results differ")


if __name__ == "__main__":
    main()
