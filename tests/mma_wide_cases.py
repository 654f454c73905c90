"""The inputs whose wide-tile outputs are pinned by SHA-256 digest in tests/golden/mma_wide_digests.json: the whole
8192^2 row and column blur pass, UnsharpMaskImage(0,4,1.5,0.02), ragged sizes along and across the filter axis, and
non-finite samples at 16-position block edges and at the image edges.  tools/mma_wide_digests.py writes the file;
tests/test_gpu_mma_tma.py checks it."""
from __future__ import annotations

import hashlib

import numpy as np

RAGGED = (1, 15, 16, 17, 31, 33, 48, 49)
EDGES = (0, 15, 16, 31, 32, 47, 48)


def rgba(w: int, h: int, seed: int) -> np.ndarray:
    """Seeded samples in [0, 65535) with about a tenth of the pixels transparent."""
    x = np.random.default_rng(seed).random((h, w, 4), dtype=np.float32) * np.float32(65535.0)
    x[..., 3] = np.where(x[..., 3] < 6553.5, np.float32(0.0), x[..., 3])
    return x


def non_finite(w: int, h: int, seed: int) -> np.ndarray:
    """rgba() with inf / -inf / NaN at block and image edges on both axes, one channel each."""
    x = rgba(w, h, seed)
    bad = (np.inf, -np.inf, np.nan)
    for i, e in enumerate(EDGES + (w - 1,)):
        x[(7 * i) % h, min(e, w - 1), i % 4] = bad[i % 3]
    for i, e in enumerate(EDGES + (h - 1,)):
        x[min(e, h - 1), (11 * i + 5) % w, (i + 1) % 4] = bad[(i + 1) % 3]
    return x


def sha256(a: np.ndarray) -> str:
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def cases():
    """(name, kind, w, h, maker): kind 'row' / 'column' is one 33-tap blur pass, 'unsharp' UnsharpMaskImage(0,4,1.5,0.02)."""
    out = [("full_row", "row", 8192, 8192, lambda: rgba(8192, 8192, 1)),
           ("full_column", "column", 8192, 8192, lambda: rgba(8192, 8192, 1)),
           ("unsharp_1031x517", "unsharp", 1031, 517, lambda: rgba(1031, 517, 2)),
           ("unsharp_4096x2048", "unsharp", 4096, 2048, lambda: rgba(4096, 2048, 3))]
    for n in RAGGED + (1031,):
        for kind in ("row", "column"):
            h = 517 if n == 1031 else 41
            out.append((f"{kind}_{n}x{h}", kind, n, h, lambda n=n, h=h: rgba(n, h, 10 + n)))
            out.append((f"{kind}_{h}x{n}", kind, h, n, lambda n=n, h=h: rgba(h, n, 20 + n)))
    for (w, h) in ((1031, 517), (49, 301), (301, 49)):
        for kind in ("row", "column", "unsharp"):
            out.append((f"nonfinite_{kind}_{w}x{h}", kind, w, h, lambda w=w, h=h: non_finite(w, h, 30 + w)))
    return out


def run(im, kind: str, src: np.ndarray):
    """The pass on the GPU; returns (output array, wide-tile launches it made)."""
    import torch
    import util
    n0 = util.get_option("conv_mma_wide_launches")
    img = im.Image(torch.from_numpy(src).cuda())
    if kind == "unsharp":
        out = im.UnsharpMaskImage(img, 0.0, 4.0, 1.5, 0.02)
    else:
        out = im.ConvolveImage(img, im.AcquireKernelInfo("blur:0x4" if kind == "row" else "blur:0x4+90"))
    got = out.pixels.cpu().numpy()
    return got, util.get_option("conv_mma_wide_launches") - n0
