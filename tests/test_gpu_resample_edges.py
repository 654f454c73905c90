"""ResizeImage, SampleImage, ScaleImage and ThumbnailImage against the oracle on the edge images of resample_edge_cases
(the oracle is pinned to the reference on the same images by test_oracle_resample_edges_vs_ref.py).

ResizeImage: NaN exactly where the oracle has NaN, the same infinities, the same zero signs, and everywhere else
within 1 ULP plus what the float intermediate's rounding can cause (cancellation_allowance): about one more ULP without
cancellation, two float ULPs of the terms where the samples cancel.  Every case runs under every forced configuration of the
run-time options -- the streaming passes with the TMA and the cp.async horizontal ring, the regular and gather kernels
of resize.cu (the regular one along x too), and the fused kernel -- and the resize_*_launches counters must show the
families a model of the table planner (plan_axis in resize_tables.cpp, fed the product's own contribution lists)
predicts, so that no case can pass on another path.  Where the fused kernel runs it must give the two streaming passes' bits; where the two factors differ by one
double ULP a forced fused launch must decline.  SampleImage and ScaleImage must be bit exact, zero signs included.
ThumbnailImage is checked stage by stage on the product's own intermediates."""
import ctypes as C
from collections import Counter

import numpy as np
import pytest

import resample_edge_cases as rc
import util
from util import P, oracle

pytestmark = pytest.mark.gpu

im = pytest.importorskip("imagemagick_b200")
torch = pytest.importorskip("torch")

FAMILIES = ("resize_fused_launches", "resize_v_stream_launches", "resize_h_tma_launches", "resize_h_stream_launches",
            "resize_regular_launches", "resize_gather_launches")
STREAMED = set(rc.SERVED.values())                                # launch_resize_stream / launch_resize_fused
# launch_regular_ch; a launcher that stops serving a pair fails the launch counters of the cases that reach it
REGULAR = {(2, 12), (2, 8), (2, 4), (3, 18), (4, 24), (4, 16)}
MAX_SEGMENTS = 8                                                  # MB200_RESIZE_MAX_SEGMENTS
# forced paths: {option: value}
CONFIGS = {
    "stream tma": {"resize_tma": 1, "no_resize_stream": 0, "no_resize_fused": 1, "resize_fused": 0, "resize_regular_h": 0},
    "stream cp.async": {"resize_tma": 0, "no_resize_stream": 0, "no_resize_fused": 1, "resize_fused": 0,
                        "resize_regular_h": 0},
    "regular v + gather h": {"resize_tma": 1, "no_resize_stream": 1, "no_resize_fused": 1, "resize_fused": 0,
                             "resize_regular_h": 0},
    "regular": {"resize_tma": 1, "no_resize_stream": 1, "no_resize_fused": 1, "resize_fused": 0, "resize_regular_h": 1},
    "fused": {"resize_tma": 1, "no_resize_stream": 0, "no_resize_fused": 0, "resize_fused": 1, "resize_regular_h": 0},
}


# ---- the planner model
_axes = {}


def axis_plan(filt, in_n, out_n, factor):
    """(stride, taps) of the regular pattern or None, the number of streamed runs, and the widest source span of an
    aligned block of 32 outputs: plan_axis over mb200_resize_contributions_ex."""
    key = (filt, in_n, out_n, factor)
    if key in _axes:
        return _axes[key]
    from imagemagick_b200 import _lib
    lib = _lib.load()
    taps = lib.mb200_resize_contributions_ex(filt, None, in_n, out_n, factor, None, None, None, 0)
    assert taps > 0, (filt, in_n, out_n)
    start, count, w = (C.c_long * out_n)(), (C.c_int * out_n)(), (C.c_double * (out_n * taps))()
    assert lib.mb200_resize_contributions_ex(filt, None, in_n, out_n, factor, start, count, w, taps) == taps
    start, count = list(start), list(count)
    w = np.ctypeslib.as_array(w).reshape(out_n, taps)
    span = max(max(start[k] + count[k] for k in range(o, min(o + 32, out_n))) - start[o] for o in range(0, out_n, 32))
    reg, nseg = None, 0
    if out_n >= 64:
        mid = out_n // 2
        n, st = count[mid], start[mid + 1] - start[mid]
        regular = sum(count[o] == n and count[o + 1] == n and start[o + 1] - start[o] == st for o in range(out_n - 1))
        if st >= 2 and n > 0 and regular * 10 >= out_n * 9:
            reg = (st, n)
            runs, lo = [], 0
            for o in range(1, out_n + 1):
                same = (o < out_n and count[o] == n and count[lo] == n and start[o] - start[o - 1] == st and
                        w[o, :n].tobytes() == w[lo, :n].tobytes())
                if not same:
                    if count[lo] == n and o - lo >= 8:
                        runs.append(o - lo)
                    lo = o
            runs = sorted(runs, reverse=True)[:MAX_SEGMENTS]
            if runs and sum(runs) * 10 >= out_n * 6:
                nseg = len(runs)
    _axes[key] = (reg, nseg, span)
    return _axes[key]


def resolved_filter(w, h, ow, oh, ch, filt):
    """resize_choice (api.cu): the factors and ResizeImage's default filter (resize.c:3804-3816)."""
    xf, yf = ow * (1.0 / w), oh * (1.0 / h)
    if filt == 0:
        filt = 1 if (xf == 1.0 and yf == 1.0) else 12 if (ch in (2, 4) or xf * yf > 1.0) else 22
    return xf, yf, filt


def expected_families(w, h, ch, ow, oh, filt, opts):
    """Counter of the resize_*_launches one ResizeImage call adds under the options `opts`."""
    if ow == w and oh == h and filt == 0:
        return Counter()                                             # a clone
    xf, yf, f = resolved_filter(w, h, ow, oh, ch, filt)
    tx, ty = axis_plan(f, w, ow, xf), axis_plan(f, h, oh, yf)
    streamed = lambda t: ch == 4 and not opts["no_resize_stream"] and t[1] > 0 and t[0] in STREAMED   # noqa: E731
    if (ch == 4 and xf == yf and not opts["no_resize_stream"] and not opts["no_resize_fused"] and opts["resize_fused"]
            and streamed(tx) and streamed(ty) and tx[0] == ty[0]):
        return Counter({"resize_fused_launches": 1})

    def one(axis, t):
        if streamed(t):
            return "resize_v_stream_launches" if axis == 1 else \
                "resize_h_tma_launches" if opts["resize_tma"] else "resize_h_stream_launches"
        if (axis == 1 or opts["resize_regular_h"]) and t[0] in REGULAR and \
                (axis == 1 or 32 * (t[2] | 1) * ch * 4 <= 48 * 1024):
            return "resize_regular_launches"
        return "resize_gather_launches"
    return Counter([one(0, tx), one(1, ty)])


# ---- comparisons
QS = 1.0 / 65535.0


def _weights(filt, in_n, out_n, factor):
    """The product's contribution lists of one axis as a dense (out_n, in_n) matrix."""
    from imagemagick_b200 import _lib
    lib = _lib.load()
    taps = lib.mb200_resize_contributions_ex(filt, None, in_n, out_n, factor, None, None, None, 0)
    start, count, w = (C.c_long * out_n)(), (C.c_int * out_n)(), (C.c_double * (out_n * taps))()
    assert lib.mb200_resize_contributions_ex(filt, None, in_n, out_n, factor, start, count, w, taps) == taps
    w = np.ctypeslib.as_array(w).reshape(out_n, taps)
    m = np.zeros((out_n, in_n))
    for o in range(out_n):
        m[o, start[o]:start[o] + count[o]] = w[o, :count[o]]
    return m


def cancellation_allowance(src, ow, oh, filt, want):
    """Per output sample, the error beyond one ULP of the result that rounding the float intermediate can cause.

    Two passes are separable: out = Wy P Wx^T for a plain channel, and (Wy (A P) Wx^T) / (Wy A Wx^T) for a colour
    blended by alpha A (the intermediate's a' p' is Wy A P exactly).  Each intermediate sample is rounded to float, so a
    kernel and the reference that differ there by one float ULP move the result by up to 2^-23 of the terms' magnitude
    M = |Wy| |P| |Wx|^T (blended: |Wy| |A P| |Wx|^T / |Wy A Wx^T| plus the alpha sum's share).  Without cancellation M
    is about |out|, so this adds at most about one ULP (an intermediate in a higher binade than the result); where the
    samples themselves cancel -- Wy |P| Wx^T exceeds twice |Wy P Wx^T| (blended: the same for A P or for A, or an alpha
    sum below PerceptibleReciprocal's threshold) -- M is far larger than |out| and the allowance is 2^-22 M, two float
    ULPs of the terms."""
    h, w, ch = src.shape
    xf, yf, f = resolved_filter(w, h, ow, oh, ch, filt)
    wy, wx = _weights(f, h, oh, yf), _weights(f, w, ow, xf)
    ay, ax = np.abs(wy), np.abs(wx)
    x = np.where(np.isfinite(src), src, 0).astype(np.float64)
    out = np.zeros(want.shape)
    cancels = lambda v: np.abs(wy @ np.abs(v) @ wx.T) > 2.0 * np.abs(wy @ v @ wx.T)   # noqa: E731
    for c in range(ch):
        target = np.abs(np.where(np.isfinite(want[..., c]), want[..., c], 0).astype(np.float64))
        with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
            if ch in (2, 4) and c < ch - 1:
                alpha, ap = x[..., ch - 1], x[..., ch - 1] * x[..., c]
                den = QS * (wy @ alpha @ wx.T)
                clamped = ~(np.abs(den) >= 1e-12)                       # PerceptibleReciprocal (resize.c:3522)
                gain = np.where(clamped, 1e12, 1.0 / np.abs(den))
                m = gain * QS * (ay @ np.abs(ap) @ ax.T)
                m += np.where(clamped, 0.0, target * gain * QS * (ay @ np.abs(alpha) @ ax.T))
                gate = clamped | cancels(ap) | cancels(alpha)
            else:
                m = ay @ np.abs(x[..., c]) @ ax.T
                gate = cancels(x[..., c])
            out[..., c] = np.where(gate, 2.0 ** -22 * m, 2.0 ** -23 * m)
    return out


def resize_disagreement(got, want, what, allowance=None):
    """None, or what differs from the oracle: NaN where the oracle has NaN, the same infinities, the same zero signs,
    and within 1 ULP plus `allowance` (cancellation_allowance) everywhere else.  Where a sum cancels, the
    kernels' FMA order (premultiplied samples, fused multiply-adds) and the reference's multiply-then-add agree to the
    last bit of the terms, not of a sum far smaller than them (+-3.4e38 under equal weights leaves a residue of ~1e20;
    a float intermediate one ULP apart moves a small HDR result by several of its own ULPs)."""
    assert got.shape == want.shape, what
    nan = np.isnan(want)
    bad = np.isnan(got) != nan
    inf = np.isinf(want)
    bad |= ~nan & (np.isinf(got) | inf) & (got != want)
    zero = (want == 0) & (got == 0)
    bad |= zero & (np.signbit(got) != np.signbit(want))
    fin = ~nan & ~inf & ~zero & np.isfinite(got)
    d = util.ulp_distance(np.where(fin, got, 0).astype(np.float32), np.where(fin, want, 0).astype(np.float32))
    near = d > 1
    if allowance is not None:
        with np.errstate(over="ignore", invalid="ignore"):            # spacing(FLT_MAX) overflows: its ULP is 2^104
            one_ulp = np.minimum(np.spacing(np.abs(np.where(fin, want, 0)).astype(np.float32)).astype(np.float64), 2.0 ** 104)
            near &= ~(np.abs(got.astype(np.float64) - want.astype(np.float64)) <= one_ulp + allowance)
    bad |= fin & near
    if not bad.any():
        return None
    at = [tuple(int(i) for i in a) for a in np.argwhere(bad)[:4]]
    return (f"{what}: {int(bad.sum())} of {bad.size} samples differ (max {int(d[fin].max()) if fin.any() else 0} ULP); "
            f"(index, got, oracle): {[(a, float(got[a]), float(want[a])) for a in at]}")


def resize_agrees(got, want, what, allowance=None):
    msg = resize_disagreement(got, want, what, allowance)
    if msg:
        pytest.fail(msg)


def report(failures):
    if failures:
        pytest.fail(f"{len(failures)} failures:\n" + "\n".join(failures[:40]))


def same_bits(got, want, what):
    """Bit-identical (zero signs included), except that any NaN matches any NaN."""
    assert got.shape == want.shape, what
    nan = np.isnan(want)
    g, w = np.where(nan, np.float32(0), got), np.where(nan, np.float32(0), want)
    bad = (np.isnan(got) != nan) | (g.view(np.int32) != w.view(np.int32))
    if bad.any():
        at = [tuple(int(i) for i in a) for a in np.argwhere(bad)[:6]]
        pytest.fail(f"{what}: {int(bad.sum())} of {bad.size} samples differ; (index, got, oracle): "
                    f"{[(a, float(got[a]), float(want[a])) for a in at]}")


def orc(name, src, ow, oh, *args):
    h, w, ch = src.shape
    out = np.full((oh, ow, ch), -12345.5, np.float32)
    assert getattr(oracle(), "orc_" + name)(P(src), w, h, ch, P(out), ow, oh, *args) == 0, (name, src.shape, ow, oh)
    return out


def _dev(a):
    return im.Image(torch.from_numpy(np.ascontiguousarray(a)).cuda())


def _host(img):
    return img.pixels.cpu().numpy() if img.on_device else img.pixels


def run_configs(src, ow, oh, filt, want, what, failures):
    """Resizes under every forced configuration, appending what differs to `failures` -- launch counters that are not
    the planned ones included, also where an option is planned to change nothing; -> {config: (output, families)}."""
    h, w, ch = src.shape
    allowance = cancellation_allowance(src, ow, oh, filt, want)
    d = _dev(src)
    outs = {}
    for name, opts in CONFIGS.items():
        expect = expected_families(w, h, ch, ow, oh, filt, opts)
        for k, v in opts.items():
            util.set_option(k, v)
        c0 = {f: util.get_option(f) for f in FAMILIES}
        got = _host(im.ResizeImage(d, ow, oh, filt))
        counts = Counter({f: util.get_option(f) - c0[f] for f in FAMILIES if util.get_option(f) != c0[f]})
        if counts != expect:
            failures.append(f"{what} [{name}]: ran {dict(counts)}, planned {dict(expect)}")
        msg = resize_disagreement(got, want, f"{what} [{name}]", allowance)
        if msg:
            failures.append(msg)
        outs[name] = (got, expect)
    return outs


# ---- ResizeImage
@pytest.mark.parametrize("ch", [1, 2, 3, 4])
def test_resize_edges(ch):
    failures = []
    for name, src, ow, oh, f in rc.resize_cases(ch):
        h, w, _ = src.shape
        outs = run_configs(src, ow, oh, f, orc("resize", src, ow, oh, f), f"{ch} {name} {w}x{h}->{ow}x{oh}", failures)
        if "fused" in outs and outs["fused"][1]["resize_fused_launches"]:
            a, b = outs["fused"][0], outs["stream tma"][0]
            if not np.array_equal(np.where(np.isnan(a), 0, a).view(np.int32), np.where(np.isnan(b), 0, b).view(np.int32)):
                failures.append(f"{ch} {name}: the fused kernel's bits differ from the two passes'")
    got = _host(im.ResizeImage(im.Image(rc.dense(ch).copy()), 18, 11, 22))          # the host entry point
    want = orc("resize", rc.dense(ch), 18, 11, 22)
    msg = resize_disagreement(got, want, f"{ch} dense host", cancellation_allowance(rc.dense(ch), 18, 11, 22, want))
    report(failures + ([msg] if msg else []))


@pytest.mark.parametrize("ch", [1, 2, 3, 4])
@pytest.mark.parametrize("case", list(rc.NAMED))
def test_named_reproductions(case, ch):
    """The signed-zero blocks: the streamed and fused kernels seeded each accumulator with its first product, so a
    window of -0 products gave -0 where the reference's sum from 0.0 gives +0."""
    build, ow, oh, f = rc.NAMED[case]
    src = build(ch)
    failures = []
    run_configs(src, ow, oh, f, orc("resize", src, ow, oh, f), f"{ch} {case}", failures)
    report(failures)


def test_every_family_is_exercised():
    """The cases above reach every resize kernel family."""
    seen = Counter()
    for name, src, ow, oh, f in rc.resize_cases(4):
        h, w, ch = src.shape
        for opts in CONFIGS.values():
            seen.update(expected_families(w, h, ch, ow, oh, f, opts))
    assert all(seen[f] > 0 for f in FAMILIES), seen


@pytest.mark.parametrize("filt", [3, 22])
def test_forced_fused_launch_declines_on_factors_one_ulp_apart(filt):
    """resize_fused=1 runs the fused kernel on equal factors (744 x 518 -> 372 x 259) and declines where the two factors
    differ by one double ULP (748 x 518 -> 374 x 259: x_factor < y_factor; 746 x 748 -> 373 x 374: x_factor > y_factor):
    there the two streaming passes run, in the reference's order, with the bits they give unforced."""
    for (w, h), (ow, oh), fused in [((744, 518), (372, 259), 1), ((748, 518), (374, 259), 0), ((746, 748), (373, 374), 0)]:
        assert (ow * (1.0 / w) == oh * (1.0 / h)) == bool(fused)
        d = _dev(rc.sparse(4, w, h, seed=13))
        runs = {}
        for name in ("fused", "stream tma"):
            for k, v in CONFIGS[name].items():
                util.set_option(k, v)
            c0 = {f: util.get_option(f) for f in FAMILIES}
            runs[name] = _host(im.ResizeImage(d, ow, oh, filt))
            counts = {f: util.get_option(f) - c0[f] for f in FAMILIES}
            assert counts["resize_gather_launches"] == counts["resize_regular_launches"] == 0, (w, h, name, counts)
            if name == "fused" and fused:
                assert counts["resize_fused_launches"] == 1 and counts["resize_v_stream_launches"] == 0, (w, h, counts)
            else:
                assert counts["resize_fused_launches"] == 0, (w, h, name, counts)
                assert counts["resize_v_stream_launches"] == counts["resize_h_tma_launches"] == 1, (w, h, name, counts)
        same_bits(runs["fused"], runs["stream tma"], f"{w}x{h} -> {ow}x{oh} forced fused against the two passes")


# ---- SampleImage, ScaleImage
@pytest.mark.parametrize("ch", [1, 2, 3, 4])
@pytest.mark.parametrize("op", ["sample", "scale"])
def test_sample_and_scale_edges(op, ch):
    fn = {"sample": im.SampleImage, "scale": im.ScaleImage}[op]
    for name, src, ow, oh in rc.sample_cases(ch):
        want = orc(op, src, ow, oh)
        same_bits(_host(fn(_dev(src), ow, oh)), want, f"{op} {ch} {name} device")
        same_bits(fn(im.Image(src.copy()), ow, oh).pixels, want, f"{op} {ch} {name} host")


# ---- ThumbnailImage
@pytest.mark.parametrize("ch", [1, 2, 3, 4])
def test_thumbnail_edges(ch):
    """The cascade stage by stage, as test_gpu_parity.test_thumbnail_pixel_path: SampleImage to 4x the target when both
    integer factors exceed 4 (bit exact), ResizeImage(Box) to 2x when they exceed 2, then ResizeImage(LanczosSharp), each
    resize stage checked against the oracle on the product's own input to it."""
    for name, src, ow, oh in rc.thumbnail_cases(ch):
        h, w, _ = src.shape
        got = _host(im.ThumbnailImage(_dev(src), ow, oh))
        if (ow, oh) == (w, h):
            same_bits(got, src, f"{ch} {name} clone")
            continue
        cur = src
        if w // ow > 4 and h // oh > 4:
            nxt = _host(im.SampleImage(_dev(cur), 4 * ow, 4 * oh))
            same_bits(nxt, orc("sample", cur, 4 * ow, 4 * oh), f"{ch} {name} sample stage")
            cur = nxt
        if w // ow > 2 and h // oh > 2:
            nxt = _host(im.ResizeImage(_dev(cur), 2 * ow, 2 * oh, im.BoxFilter))
            want = orc("resize", cur, 2 * ow, 2 * oh, 2)
            resize_agrees(nxt, want, f"{ch} {name} box stage", cancellation_allowance(cur, 2 * ow, 2 * oh, 2, want))
            cur = nxt
        same_bits(got, _host(im.ResizeImage(_dev(cur), ow, oh, im.LanczosSharpFilter)), f"{ch} {name} cascade")
        cur = np.ascontiguousarray(cur)
        want = orc("resize", cur, ow, oh, 23)
        resize_agrees(got, want, f"{ch} {name} last stage", cancellation_allowance(cur, ow, oh, 23, want))
