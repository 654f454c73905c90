"""The oracle of the last three image-returning accelerate hooks -- DespeckleImage (effect.c:1308), LocalContrastImage
(effect.c:2013) and WaveletDenoiseImage (visual-effects.c:3515) -- against the reference, bit for bit.

The oracle is oracle/hooks_oracle.c (oracle/libhooks_oracle.so) and the reference driver oracle/ref_hooks.c
(oracle/_ref/libmagickref_hooks.so), both built by oracle/Makefile.  What the reference computed for every case is stored
as a digest (util.digest) in tests/golden/hook_digests.json, keyed like util.reference keys tests/golden/ref_digests.json;
re-record it with MB200_RECORD_REFERENCE=1 where oracle/_ref is built."""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

import util
from util import P, ROOT, digest, make_image

_fp, _sz, _d, _i = C.POINTER(C.c_float), C.c_size_t, C.c_double, C.c_int
ORACLE_SO = ROOT / "oracle" / "libhooks_oracle.so"
REF_SO = ROOT / "oracle" / "_ref" / "libmagickref_hooks.so"
DIGESTS = ROOT / "tests" / "golden" / "hook_digests.json"
_libs = {}


def oracle():
    """The plain-C oracle; (re)built when stale, like conftest.py does for oracle/liboracle.so."""
    if "oracle" not in _libs:
        o = util.load_oracle(ORACLE_SO)
        o.orc_despeckle.argtypes = [_fp, _fp, _sz, _sz, _i]
        o.orc_local_contrast.argtypes = [_fp, _fp, _sz, _sz, _i, _d, _d]
        o.orc_wavelet_denoise.argtypes = [_fp, _fp, _sz, _sz, _i, _d, _d]
        _libs["oracle"] = o
    return _libs["oracle"]


def ref():
    """The real reference's operators; only where oracle/_ref has been built from a reference source tree."""
    if "ref" not in _libs:
        r = C.CDLL(str(REF_SO))
        r.ref_despeckle.argtypes = [_fp, _fp, _sz, _sz, _i]
        r.ref_local_contrast.argtypes = [_fp, _fp, _sz, _sz, _i, _d, _d]
        r.ref_wavelet_denoise.argtypes = [_fp, _fp, _sz, _sz, _i, _d, _d, _i]
        _libs["ref"] = r
    return _libs["ref"]


_store = util.ReferenceStore(DIGESTS, REF_SO)


def reference(case: str, run):
    """Digest of what the reference computed for `case` of the running test: of the output array run() returns with
    the reference itself when recording."""
    return _store(case, lambda: digest(run()))


def hook_image(w, h, ch, kind, seed=5):
    """make_image's kinds plus `posterised`: few levels, multiples of 257 (Despeckle's steps: its comparisons tie)
    and `black`: noise with some pixels 0 in every channel (LocalContrast's luma-0 pixels, NaN in the reference)."""
    if kind == "posterised":
        rng = np.random.default_rng(seed)
        a = (rng.integers(100, 106, (h, w, ch)) * 257).astype(np.float32)
        return np.ascontiguousarray(a)
    a = make_image(w, h, ch, seed=seed, kind="noise" if kind == "black" else kind)
    if kind == "black":
        a[::5, ::3, :] = 0.0
    return a


def run(fn, src, *args):
    h, w, ch = src.shape
    out = np.full_like(src, -7.0)
    rc = fn(P(src), P(out), w, h, ch, *args)
    return out if rc == 0 else np.array([rc], np.float32)


def oracle_despeckle(src):
    return run(oracle().orc_despeckle, src)


def oracle_local_contrast(src, radius, strength):
    return run(oracle().orc_local_contrast, src, radius, strength)


def oracle_wavelet(src, threshold, softness):
    return run(oracle().orc_wavelet_denoise, src, threshold, softness)


KINDS = ["noise", "alpha_blocks", "hdr", "posterised"]


@pytest.mark.parametrize("ch", [1, 2, 3, 4])
@pytest.mark.parametrize("kind", KINDS)
def test_despeckle_bit_exact(ch, kind):
    for w, h in [(37, 23), (19, 41), (1, 17), (23, 1), (2, 2)]:
        src = hook_image(w, h, ch, kind)
        b = oracle_despeckle(src)
        assert b.shape == src.shape
        assert digest(b) == reference(f"{w}x{h}", lambda: run(ref().ref_despeckle, src)), (w, h)


def test_despeckle_changes_posterised_pixels():
    """The posterised cases are not trivial: the hulls move values by 257 steps there."""
    src = hook_image(37, 23, 3, "posterised")
    assert (oracle_despeckle(src) != src).mean() > 0.1


@pytest.mark.parametrize("ch", [1, 2, 3, 4])
@pytest.mark.parametrize("kind", ["noise", "alpha_blocks", "hdr", "posterised", "black"])
def test_local_contrast_bit_exact(ch, kind):
    cases = [(61, 47, 0.0, 12.5), (61, 47, 10.0, 12.5), (61, 47, 40.0, -40.0), (61, 47, 100.0, 100.0),
             (61, 47, 250.0, 0.0), (61, 47, 491.0, 12.5), (23, 67, 164.0, 60.0), (23, 67, -20.0, -12.5)]
    for w, h, radius, strength in cases:
        src = hook_image(w, h, ch, kind)
        b = oracle_local_contrast(src, radius, strength)
        assert b.shape == src.shape, (w, h, radius)
        assert digest(b) == reference(f"{w}x{h},{radius},{strength}",
                                      lambda: run(ref().ref_local_contrast, src, radius, strength)), (w, h, radius, strength)


def test_local_contrast_black_pixels_are_nan():
    src = hook_image(61, 47, 3, "black")
    b = oracle_local_contrast(src, 10.0, 12.5)
    black = (src == 0).all(axis=2)
    assert np.isnan(b[black]).all() and not np.isnan(b[~black]).any()


def test_local_contrast_width_bound():
    """The mirror padding covers width <= columns - 1; one more and the reference reads what it never wrote."""
    src = hook_image(61, 47, 3, "noise")
    # width = (ssize_t) (61 * 0.002 * radius): 60 at radius 492, 61 at radius 500
    assert oracle_local_contrast(src, 492.0, 12.5).shape == src.shape
    assert oracle_local_contrast(src, 500.0, 12.5).shape == (1,)
    tall = hook_image(3, 600, 1, "noise")              # width = (ssize_t) (600 * 0.002 * 2) = 2 = columns - 1
    assert oracle_local_contrast(tall, 2.0, 12.5).shape == tall.shape
    assert oracle_local_contrast(tall, 2.5, 12.5).shape == (1,)


@pytest.mark.parametrize("ch", [1, 2, 3, 4])
@pytest.mark.parametrize("kind", KINDS)
def test_wavelet_denoise_bit_exact(ch, kind):
    cases = [(32, 32, 0.0, 0.0), (33, 45, 500.0, 0.0), (45, 32, 500.0, 0.3), (64, 37, 6553.5, 1.0),
             (37, 64, 6553.5, 0.3), (40, 33, 20000.0, 0.0)]
    for w, h, threshold, softness in cases:
        src = hook_image(w, h, ch, kind)
        b = oracle_wavelet(src, threshold, softness)
        assert b.shape == src.shape
        assert digest(b) == reference(f"{w}x{h},{threshold},{softness}",
                                      lambda: run(ref().ref_wavelet_denoise, src, threshold, softness, 0)), \
            (w, h, threshold, softness)


@pytest.mark.parametrize("ch", [3, 4])
def test_wavelet_denoise_ignores_the_channel_selection(ch):
    """The reference's loop tests only for an Undefined trait (visual-effects.c:3607-3614), so a `-channel` selection
    (Copy traits on the unselected channels) changes nothing: red, green and blue are all denoised."""
    src = hook_image(41, 35, ch, "noise")
    b = oracle_wavelet(src, 3000.0, 0.3)
    for mask in (0x1, 0x10 | 0x1):                      # RedChannel, Red + Alpha
        assert digest(b) == reference(f"{mask}", lambda: run(ref().ref_wavelet_denoise, src, 3000.0, 0.3, mask)), mask


def test_wavelet_denoise_size_bound():
    """The level-4 hat (step 16) needs 32 samples per line; below that HatTransform reads outside the line."""
    for w, h in [(31, 40), (40, 31), (31, 31)]:
        assert oracle_wavelet(hook_image(w, h, 3, "noise"), 500.0, 0.0).shape == (1,), (w, h)
    assert oracle_wavelet(hook_image(32, 32, 3, "noise"), 500.0, 0.0).shape == (32, 32, 3)
