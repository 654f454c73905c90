"""Test helpers: ctypes access to the oracle (tests only!), ULP metrics, fixtures."""
from __future__ import annotations

import atexit
import ctypes as C
import hashlib
import json
import os
import subprocess
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
ORACLE_SO = ROOT / "oracle" / "liboracle.so"
REF_SO = ROOT / "oracle" / "_ref" / "libmagickref.so"
REF_DIGESTS = ROOT / "tests" / "golden" / "ref_digests.json"

_fp = C.POINTER(C.c_float)
_sz, _d, _i, _l = C.c_size_t, C.c_double, C.c_int, C.c_long


def P(a: np.ndarray):
    assert a.dtype == np.float32 and a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(_fp)


class OrcKernel(C.Structure):
    _fields_ = [("width", _sz), ("height", _sz), ("x", _l), ("y", _l), ("values", C.POINTER(_d)),
                ("minimum", _d), ("maximum", _d), ("negative_range", _d), ("positive_range", _d), ("type", _i)]

    def array(self):
        n = self.width * self.height
        return np.array([self.values[i] for i in range(n)]).reshape(self.height, self.width)


# oracle kernel type ids (oracle.h)
ORC_K = dict(blur=0, gaussian=1, disk=2, square=3, diamond=4, octagon=5, plus=6, cross=7, rectangle=8)

_oracle = None
_ref = None


def oracle() -> C.CDLL:
    global _oracle
    if _oracle is None:
        o = C.CDLL(str(ORACLE_SO))
        for f in (o.orc_blur, o.orc_gaussian_blur):
            f.argtypes = [_fp, _fp, _sz, _sz, _i, _d, _d]
        o.orc_unsharp.argtypes = [_fp, _fp, _sz, _sz, _i, _d, _d, _d, _d]
        o.orc_sharpen.argtypes = [_fp, _fp, _sz, _sz, _i, _d, _d]
        o.orc_motion_blur.argtypes = [_fp, _fp, _sz, _sz, _i, _d, _d, _d]
        o.orc_bilateral_blur.argtypes = [_fp, _fp, _sz, _sz, _i, _sz, _sz, _d, _d]
        o.orc_rotational_blur.argtypes = [_fp, _fp, _sz, _sz, _i, _d]
        o.orc_statistic.argtypes = [_fp, _fp, _sz, _sz, _i, _i, _sz, _sz]
        o.orc_edge.argtypes = [_fp, _fp, _sz, _sz, _i, _d]
        o.orc_emboss.argtypes = [_fp, _fp, _sz, _sz, _i, _d, _d]
        o.orc_emboss_kernel.argtypes = [_d, _d, C.POINTER(OrcKernel)]
        o.orc_equalize.argtypes = [_fp, _sz, _sz, _i, _i]
        o.orc_resize.argtypes = [_fp, _sz, _sz, _i, _fp, _sz, _sz, _i]
        o.orc_resize_ex.argtypes = [_fp, _sz, _sz, _i, _fp, _sz, _sz, _i, C.c_void_p]
        o.orc_filter_weight_ex.argtypes = [_i, C.c_void_p, _d]
        o.orc_filter_weight_ex.restype = _d
        o.orc_filter_support_ex.argtypes = [_i, C.c_void_p]
        o.orc_filter_support_ex.restype = _d
        o.orc_colorspace.argtypes = [_fp, _sz, _sz, _i, _i, _i]
        o.orc_colorspace_ex.argtypes = [_fp, _sz, _sz, _i, _i, _i, C.c_void_p]
        o.orc_log_table.argtypes = [_i, C.c_void_p, _fp]
        o.orc_log_table.restype = None
        o.orc_ycc_table.argtypes = [_fp]
        o.orc_ycc_table.restype = None
        o.orc_sample.argtypes = [_fp, _sz, _sz, _i, _fp, _sz, _sz]
        o.orc_scale.argtypes = [_fp, _sz, _sz, _i, _fp, _sz, _sz]
        o.orc_selective_blur.argtypes = [_fp, _fp, _sz, _sz, _i, _d, _d, _d]
        o.orc_adaptive_blur.argtypes = [_fp, _fp, _sz, _sz, _i, _d, _d]
        o.orc_adaptive_sharpen.argtypes = [_fp, _fp, _sz, _sz, _i, _d, _d]
        o.orc_thumbnail.argtypes = [_fp, _sz, _sz, _i, _fp, _sz, _sz]
        o.orc_kernel_builtin.argtypes = [_i, _d, _d, _d, _d, C.POINTER(OrcKernel)]
        o.orc_kernel_user.argtypes = [_sz, _sz, _l, _l, C.POINTER(_d), C.POINTER(OrcKernel)]
        o.orc_kernel_free.argtypes = [C.POINTER(OrcKernel)]
        o.orc_morphology_apply.argtypes = [_fp, _fp, _sz, _sz, _i, _i, _l, C.POINTER(OrcKernel), _i, _d]
        o.orc_morphology_primitive.argtypes = [_fp, _fp, _sz, _sz, _i, _i, C.POINTER(OrcKernel), _d]
        o.orc_morphology_primitive.restype = _l
        o.orc_filter_weight.argtypes = [_i, _d]
        o.orc_filter_weight.restype = _d
        o.orc_filter_support.argtypes = [_i]
        o.orc_filter_support.restype = _d
        o.orc_optimal_kernel_width_1d.argtypes = [_d, _d]
        o.orc_optimal_kernel_width_1d.restype = _sz
        o.orc_optimal_kernel_width_2d.argtypes = [_d, _d]
        o.orc_optimal_kernel_width_2d.restype = _sz
        o.orc_threshold.argtypes = [_fp, _sz, _sz, _i, _i, C.POINTER(_d)]
        o.orc_set_threads.argtypes = [_i]
        _oracle = o
    return _oracle


_port_built = False


def load_oracle(path: Path) -> C.CDLL:
    """The plain-C oracle library `path` (oracle/lib*.so), once `make port` has brought every oracle library up to date
    (run once per process: make decides what is stale)."""
    global _port_built
    if not _port_built:
        env = dict(os.environ)
        env.pop("CC", None)
        subprocess.run(["make", "-s", "-C", str(ROOT / "oracle"), "port"], check=True, env=env,
                       stdout=subprocess.DEVNULL)
        _port_built = True
    return C.CDLL(str(path))


def have_ref() -> bool:
    return REF_SO.exists()


def ref() -> C.CDLL:
    """The real reference (ImageMagick compiled from source); only exists where
    oracle/_ref has been built from a reference source tree (oracle/Makefile)."""
    global _ref
    if _ref is None:
        r = C.CDLL(str(REF_SO))
        for f in (r.ref_blur, r.ref_gaussian_blur):
            f.argtypes = [_fp, _fp, _sz, _sz, _i, _d, _d]
        r.ref_unsharp.argtypes = [_fp, _fp, _sz, _sz, _i, _d, _d, _d, _d]
        r.ref_sharpen.argtypes = [_fp, _fp, _sz, _sz, _i, _d, _d]
        r.ref_motion_blur.argtypes = [_fp, _fp, _sz, _sz, _i, _d, _d, _d]
        r.ref_bilateral_blur.argtypes = [_fp, _fp, _sz, _sz, _i, _sz, _sz, _d, _d]
        r.ref_rotational_blur.argtypes = [_fp, _fp, _sz, _sz, _i, _d]
        r.ref_statistic.argtypes = [_fp, _fp, _sz, _sz, _i, _i, _sz, _sz]
        r.ref_edge.argtypes = [_fp, _fp, _sz, _sz, _i, _d]
        r.ref_emboss.argtypes = [_fp, _fp, _sz, _sz, _i, _d, _d]
        r.ref_equalize.argtypes = [_fp, _sz, _sz, _i, _i]
        r.ref_convolve.argtypes = [_fp, _fp, _sz, _sz, _i, C.c_char_p]
        r.ref_morphology.argtypes = [_fp, _fp, _sz, _sz, _i, _i, _l, C.c_char_p]
        r.ref_resize.argtypes = [_fp, _sz, _sz, _i, _fp, _sz, _sz, _i]
        r.ref_resize_defines.argtypes = [_fp, _sz, _sz, _i, _fp, _sz, _sz, _i, C.c_char_p]
        r.ref_colorspace.argtypes = [_fp, _sz, _sz, _i, _i, _i]
        r.ref_colorspace_defines.argtypes = [_fp, _sz, _sz, _i, _i, _i, C.c_char_p]
        r.ref_sample.argtypes = [_fp, _sz, _sz, _i, _fp, _sz, _sz]
        r.ref_scale.argtypes = [_fp, _sz, _sz, _i, _fp, _sz, _sz]
        r.ref_selective_blur.argtypes = [_fp, _fp, _sz, _sz, _i, _d, _d, _d]
        r.ref_adaptive_blur.argtypes = [_fp, _fp, _sz, _sz, _i, _d, _d]
        r.ref_adaptive_sharpen.argtypes = [_fp, _fp, _sz, _sz, _i, _d, _d]
        r.ref_thumbnail.argtypes = [_fp, _sz, _sz, _i, _fp, _sz, _sz]
        r.ref_kernel.argtypes = [C.c_char_p, _i, C.POINTER(_d), _sz, C.POINTER(_sz), C.POINTER(_sz),
                                 C.POINTER(_l), C.POINTER(_l)]
        r.ref_threshold.argtypes = [_fp, _sz, _sz, _i, _i, _d, C.c_char_p]
        r.ref_version.restype = C.c_char_p
        r.ref_set_threads.argtypes = [_i]
        _ref = r
    return _ref


def digest(a: np.ndarray) -> str:
    """Short SHA-256 of an array's dtype, shape and values.  Every NaN hashes as one NaN and -0 as +0, so two arrays
    have the same digest exactly when max_ulp() between them is 0 (NaN where either has NaN)."""
    a = np.ascontiguousarray(a)
    if a.dtype.kind == "f":
        a = np.where(np.isnan(a), np.array(np.nan, a.dtype), a + a.dtype.type(0))
    h = hashlib.sha256(f"{a.dtype.str}{a.shape}".encode())
    h.update(a.tobytes())
    return h.hexdigest()[:10]


def current_test() -> str:
    """The running test as "<file>::<test>[<parameter id>]": its node id without the directory and the phase."""
    test = os.environ.get("PYTEST_CURRENT_TEST", "").rsplit(" (", 1)[0].split("::", 1)
    return test[0].rsplit("/", 1)[-1] + "::" + test[-1]


def zero_signs(a: np.ndarray) -> str:
    """Digest of where the zeros of `a` are negative: digest() hashes -0 as +0, so this pins the sign of a zero."""
    return digest((a == 0) & np.signbit(a))


class ReferenceStore:
    """What the reference computed, stored as strings in the JSON file `path`: nested as {"<file>::<test>[<params>]":
    {case: value}} (by_test, the running test's or `test`'s entries) or flat as {case: value}.

    store(case, run, test=None) returns the stored value and asserts there is one.  With MB200_RECORD_REFERENCE=1 and
    the reference library `ref_so` built, it returns run() instead, which computes the value with the reference itself,
    and records it into `path` (merged into what is there) when the process exits."""

    def __init__(self, path: Path, ref_so: Path, by_test: bool = True):
        self.path, self.ref_so, self.by_test = path, ref_so, by_test
        self.stored = None
        self.recorded = {}

    def entries(self, test: str = None) -> dict:
        """case -> value of `test` (nested), or of the whole file (flat)."""
        if self.stored is None:
            self.stored = json.loads(self.path.read_text())
        return self.stored.get(test, {}) if self.by_test else self.stored

    def __call__(self, case: str, run, test: str = None) -> str:
        if self.by_test and test is None:
            test = current_test()
        if os.environ.get("MB200_RECORD_REFERENCE") == "1" and self.ref_so.exists():
            return self.record(case, run(), test)
        stored = self.entries(test)
        assert case in stored, "no stored reference result for " + (f"{test} / {case}" if self.by_test else case)
        return stored[case]

    def record(self, case: str, value: str, test: str = None) -> str:
        if not self.recorded:
            atexit.register(self._save)
        self.recorded[(test, case) if self.by_test else case] = value
        return value

    def _save(self):
        data = json.loads(self.path.read_text()) if self.path.exists() else {}
        if self.by_test:
            for (test, case), value in self.recorded.items():
                data.setdefault(test, {})[case] = value
            lines = (json.dumps(t) + ": " + json.dumps(c, separators=(",", ":")) for t, c in sorted(data.items()))
        else:
            data.update(self.recorded)
            lines = (json.dumps(k) + ": " + json.dumps(v) for k, v in sorted(data.items()))
        self.path.write_text("{\n" + ",\n".join(lines) + "\n}\n")


REF_STORE = ReferenceStore(REF_DIGESTS, REF_SO)


def record(group: str, case: str, a: np.ndarray) -> str:
    """Stores the digest of the reference's output `a` as `group` / `case` of tests/golden/ref_digests.json (written
    when the process exits)."""
    return REF_STORE.record(case, digest(a), group)


def stored_digests(group: str) -> dict:
    return REF_STORE.entries(group)


def reference(case: str, run):
    """Digest of what the reference computed for `case` of the running test, from tests/golden/ref_digests.json.
    With MB200_RECORD_REFERENCE=1 and oracle/_ref built, run() computes it with the reference itself (it returns the
    output array) and the digest is recorded into that file when the process exits."""
    return REF_STORE(case, lambda: digest(run()))


def ref_kernel(string: str, idx: int = 0):
    vals = (_d * 65536)()
    kw, kh, kx, ky = _sz(), _sz(), _l(), _l()
    rc = ref().ref_kernel(string.encode(), idx, vals, 65536, C.byref(kw), C.byref(kh), C.byref(kx), C.byref(ky))
    if rc:
        return None
    return np.array(vals[: kw.value * kh.value]).reshape(kh.value, kw.value), kx.value, ky.value


def orc_kernel(kind: str, rho=0.0, sigma=0.0, xi=0.0, psi=0.0) -> OrcKernel:
    k = OrcKernel()
    rc = oracle().orc_kernel_builtin(ORC_K[kind], rho, sigma, xi, psi, C.byref(k))
    assert rc == 0, (kind, rho, sigma, xi, psi)
    return k


def orc_kernel_from_array(values: np.ndarray, x: int, y: int) -> OrcKernel:
    v = np.ascontiguousarray(values, dtype=np.float64)
    k = OrcKernel()
    rc = oracle().orc_kernel_user(v.shape[1], v.shape[0], x, y, v.ctypes.data_as(C.POINTER(_d)), C.byref(k))
    assert rc == 0
    return k


def orc_morphology(src: np.ndarray, method: int, iterations: int, kernels, bias=0.0) -> np.ndarray:
    h, w, ch = src.shape
    arr = (OrcKernel * len(kernels))(*kernels)
    dst = np.empty_like(src)
    rc = oracle().orc_morphology_apply(P(src), P(dst), w, h, ch, method, iterations, arr, len(kernels), bias)
    assert rc == 0
    return dst


def ulp_distance(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    """Per-element distance in float32 ULPs (sign-magnitude ordered integers)."""
    assert a.shape == b.shape and a.dtype == np.float32 and b.dtype == np.float32
    ai = a.view(np.int32).astype(np.int64)
    bi = b.view(np.int32).astype(np.int64)
    ai = np.where(ai < 0, -(ai & 0x7FFFFFFF), ai)
    bi = np.where(bi < 0, -(bi & 0x7FFFFFFF), bi)
    return np.abs(ai - bi)


def max_ulp(a, b) -> int:
    return int(ulp_distance(np.ascontiguousarray(a), np.ascontiguousarray(b)).max())


class FilterOptions(C.Structure):
    """mb200_filter_options == orc_filter_options: the "filter:*" expert settings as values."""
    _fields_ = [("set", C.c_uint), ("window", C.c_int), ("keep_filter", C.c_int), ("lobes", C.c_long), ("sigma", C.c_double),
                ("kaiser_beta", C.c_double), ("blur", C.c_double), ("support", C.c_double), ("win_support", C.c_double),
                ("b", C.c_double), ("c", C.c_double)]

    BITS = {"window": 1, "sigma": 2, "kaiser_beta": 4, "lobes": 8, "blur": 16, "support": 32, "win_support": 64, "b": 128, "c": 256}

    @classmethod
    def of(cls, **kw):
        o = cls()
        for k, v in kw.items():
            if k == "keep_filter":
                o.keep_filter = int(v)
                continue
            setattr(o, k, v)
            o.set |= cls.BITS[k]
        return o


class ColorspaceOptions(C.Structure):
    """mb200_colorspace_options == orc_colorspace_options: the image settings TransformImageColorspace reads, as values."""
    _fields_ = [("set", C.c_uint), ("illuminant", C.c_int), ("white_luminance", C.c_double),
                ("film_gamma", C.c_double), ("reference_black", C.c_double), ("reference_white", C.c_double)]

    BITS = {"illuminant": 1, "white_luminance": 2, "film_gamma": 4, "reference_black": 8, "reference_white": 16}
    ILLUMINANTS = {"A": 0, "B": 1, "C": 2, "D50": 3, "D55": 4, "D65": 5, "D75": 6, "E": 7, "F2": 8, "F7": 9, "F11": 10}

    @classmethod
    def of(cls, **kw):
        o = cls()
        for k, v in kw.items():
            setattr(o, k, cls.ILLUMINANTS[v] if k == "illuminant" else v)
            o.set |= cls.BITS[k]
        return o


def ulp_or_noise(a, b, tiny=1.0e-6) -> np.ndarray:
    """ULP distance, except where BOTH values are rounding noise around zero (|v| < tiny Quantum units = 1.5e-11 of full
    scale): a component the reference computes as the difference of two equal numbers -- e.g. the red channel of an
    Adobe98 blue taken to sRGB, whose primaries coincide -- has no significant bits to compare; 0 is returned there."""
    d = ulp_distance(np.ascontiguousarray(a), np.ascontiguousarray(b))
    noise = (np.abs(a) < tiny) & (np.abs(b) < tiny)
    return np.where(noise, 0, d)


def frac_exact(a, b) -> float:
    return float((ulp_distance(np.ascontiguousarray(a), np.ascontiguousarray(b)) == 0).mean())


def make_image(w: int, h: int, ch: int, seed: int = 42, kind: str = "noise") -> np.ndarray:
    """Seeded synthetic pixel cache (raw Quantum floats 0..65535).
    kind: noise | alpha_blocks (fully transparent / opaque regions, exercises
    PerceptibleReciprocal) | gradient | hdr (values outside 0..QuantumRange, negatives)."""
    rng = np.random.default_rng(seed)
    a = (rng.random((h, w, ch), dtype=np.float32) * np.float32(65535.0)).astype(np.float32)
    if kind == "alpha_blocks" and ch in (2, 4):
        a[: h // 2, : w // 2, ch - 1] = 0.0
        a[h // 2:, w // 2:, ch - 1] = 65535.0
        a[h // 3: h // 3 + 2, :, ch - 1] = 1.0
    elif kind == "gradient":
        yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
        for c in range(ch):
            a[..., c] = ((xx * (c + 1) + yy * 3) % 256) * 257.0
    elif kind == "hdr":
        a = (a - 20000.0) * 1.7
    elif kind == "binary":
        a = np.where(a > 40000.0, np.float32(65535.0), np.float32(0.0)).astype(np.float32)
    return np.ascontiguousarray(a)


def parse_thresholds(spec: str):
    """The ParseGeometry step of Black/WhiteThresholdImage (threshold.c:955-985) for the
    'v[,v[,v[,v]]][%]' forms: returns [red, green, blue, alpha] in Quantum units."""
    pct = "%" in spec
    vals = [float(t) for t in spec.replace("%", "").split(",") if t.strip()]
    rho = vals[0]
    thr = [rho, vals[1] if len(vals) > 1 else rho, vals[2] if len(vals) > 2 else rho,
           vals[3] if len(vals) > 3 else 100.0]
    if pct:
        thr = [t * (65535.0 / 100.0) for t in thr]
    return thr


def orc_threshold(src: np.ndarray, op: int, thr) -> np.ndarray:
    h, w, ch = src.shape
    out = src.copy()
    arr = (_d * 4)(*([float(t) for t in thr] + [0.0] * (4 - len(thr))))
    assert oracle().orc_threshold(P(out), w, h, ch, op, arr) == 0
    return out


# ---- run-time switches of the product library (mb200_set_option): restored after every test by conftest.py
_touched_options = {}


def get_option(name: str) -> int:
    from imagemagick_b200 import _lib
    v = C.c_int(0)
    _lib.check(_lib.load().mb200_get_option(name.encode(), C.byref(v)))
    return int(v.value)


def set_option(name: str, value: int) -> None:
    from imagemagick_b200 import _lib
    if name not in _touched_options:
        _touched_options[name] = get_option(name)       # the process default (environment), restored after the test
    _lib.check(_lib.load().mb200_set_option(name.encode(), int(value)))


def reset_options() -> None:
    if not _touched_options:
        return
    from imagemagick_b200 import _lib
    for name, value in list(_touched_options.items()):
        _lib.load().mb200_set_option(name.encode(), value)
    _touched_options.clear()
