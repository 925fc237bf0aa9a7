"""The JNI shim (distributed_sgd_b200/jni/dsgd_jni.c) run against libdsgd.so through a stand-in JNIEnv (tests/jni_mock/):
Java arrays are (element type, length, data) records, and a region copy of the wrong element type is counted.  The shim's
functions get the handles of NativeCtx contexts: an SVM one, a logistic one with an intercept and an async one.

* Every native that NativeCtx also binds gives NativeCtx's result (or its error code) bit for bit; the logistic gradient
  adds with fp64 atomics in the order the rows arrive, so it agrees to rounding, as in test_gpu_request_paths.py.
* Every array the shim hands to the library is checked first: one element too short (and w one too long) is
  DSGD_ERR_INVALID, with no launch and the output arrays as they were.
* getWeights, which may run on several threads at once, gives the resident weights from eight threads."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from distributed_sgd_b200.native import weighted_auc_ap

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N_ROWS, LAM, KEY = 3000, 1e-4, 0x9E3779B97F4A7C15
N = 300                                                    # rows of one request
SIGMOID, N_BINS = (1.5, -0.25), 10
MAP = (np.array([-2.0, 0.0, 2.0]), np.array([0.2, 0.5, 0.8]))
BOOT = (3, 0, 4)                                           # bkey, [b_begin, b_end)
SENTINEL = 0x5A


class JArray(C.Structure):
    _fields_ = [("type", C.c_int32), ("n", C.c_int32), ("data", C.c_void_p)]


_JTYPE = {np.dtype(np.int32): 0, np.dtype(np.int64): 1, np.dtype(np.float32): 2, np.dtype(np.float64): 3,
          np.dtype(np.int8): 4}
_CTYPE = {"Long": C.c_int64, "Int": C.c_int32, "Double": C.c_double, "String": C.c_void_p}


def scala_natives():
    """{native: (parameter ctypes, result ctype)} from the declarations of DsgdNative.scala"""
    text = open(os.path.join(ROOT, "distributed_sgd_b200", "jni", "DsgdNative.scala")).read()
    out = {}
    for name, params, res in re.findall(r"@native def (\w+)\(([^)]*)\):\s*(\w+)", text):
        types = [p.split(":")[1].strip() for p in params.split(",")]
        out[name] = ([C.c_void_p if t.startswith("Array[") else _CTYPE[t] for t in types], _CTYPE[res])
    return out


class Shim:
    """dsgd_jni.c and the stand-in JNIEnv in one library linked against the package's libdsgd.so"""

    def __init__(self, path):
        from distributed_sgd_b200 import native
        native.lib()
        pkg = os.path.dirname(native.LIB_PATH)
        subprocess.run(["gcc", "-std=gnu11", "-Wall", "-Wextra", "-Wno-unused-parameter", "-Werror", "-shared", "-fPIC",
                        "-DDSGD_HAVE_JNI", "-I" + os.path.join(ROOT, "tests", "jni_mock"), "-I" + os.path.join(ROOT, "include"),
                        os.path.join(ROOT, "distributed_sgd_b200", "jni", "dsgd_jni.c"),
                        os.path.join(ROOT, "tests", "jni_mock", "jni_env.c"), "-L" + pkg, "-ldsgd", "-Wl,-rpath," + pkg,
                        "-o", path], check=True)
        self.lib = C.CDLL(path)
        self.lib.mock_env.restype = C.c_void_p
        self.env = self.lib.mock_env()
        self.natives = scala_natives()

    def __call__(self, name, *args):
        """rc of the native `name`; numpy arrays go in as Java arrays (their memory), None as a null array"""
        fn = getattr(self.lib, "Java_epfl_distributed_nativ_DsgdNative_00024_" + name)
        types, res = self.natives[name]
        fn.argtypes, fn.restype = [C.c_void_p, C.c_void_p] + types, res
        keep = [JArray(_JTYPE[a.dtype], a.size, a.ctypes.data) if isinstance(a, np.ndarray) else a for a in args]
        return fn(self.env, None, *[C.addressof(a) if isinstance(a, JArray) else a for a in keep])

    def region_errors(self):
        return self.lib.mock_region_errors()


def out(n, dtype):
    """an output array of n elements, every byte SENTINEL"""
    return np.full(max(int(n), 0) * np.dtype(dtype).itemsize, SENTINEL, np.uint8).view(dtype)


I64, F64 = np.int64, np.float64


def bits(x):
    if isinstance(x, (tuple, list)):
        return tuple(bits(v) for v in x)
    if isinstance(x, np.ndarray):
        return x.dtype.str, x.shape, x.tobytes()
    return float(x).hex() if isinstance(x, float) else int(x)


# The evaluation families: name -> (the arguments after the rows, the shim's output arrays for n rows, and the NativeCtx
# result rebuilt from them)
def _quality(words):
    return lambda n: [out(2, F64), out(N_BINS, I64), out(N_BINS, I64), out(N_BINS, F64), out(words, I64)]


def _wquality(words):
    return lambda n: [out(4, F64), out(N_BINS, F64), out(N_BINS, F64), out(N_BINS, F64), out(words, I64)]


def _iso_fit(o):
    k, nb = int(o[0][0]), int(o[5][0])
    return (o[1][:k], o[2][:k], o[3][:nb], o[4][:nb], o[5])


k_boot = BOOT[2] - BOOT[1]
FAMILIES = {
    "counts": ((), lambda n: [out(2, I64), out(1, F64)], lambda o: (o[0][0], o[0][1], o[1][0])),
    "sums": ((), lambda n: [out(2, F64), out(1, I64)], lambda o: (o[0][0], o[1][0], o[0][1])),
    "class": ((), lambda n: [out(3, F64), out(4, I64)], lambda o: (*o[0], *o[1])),
    "weighted": ((), lambda n: [out(4, F64), out(2, I64)], lambda o: (*o[0], *o[1])),
    "metrics": ((), lambda n: [out(8, I64)], lambda o: o[0]),
    "curve": ((), lambda n: [out(8, I64), out(1, F64), out(1, I64), out(n, F64), out(n, I64), out(n, I64)],
              lambda o: (o[0], o[1][0], o[3][:o[2][0]], o[4][:o[2][0]], o[5][:o[2][0]])),
    "weighted_curve": ((), lambda n: [out(8, I64), out(13, F64), out(1, I64), out(n, F64), out(n, F64), out(n, F64)],
                       lambda o: (o[0], o[1], o[2][0], o[3][:o[2][0]], o[4][:o[2][0]], o[5][:o[2][0]],
                                  *weighted_auc_ap(o[0], o[1]))),
    "bootstrap": (BOOT, lambda n: [out(9 * k_boot, I64), out(k_boot, F64), out(k_boot, F64)],
                  lambda o: (o[0].reshape(k_boot, 9), o[1], o[2])),
    "weighted_bootstrap": (BOOT, lambda n: [out(2 * k_boot, I64), out(13 * k_boot, F64), out(k_boot, F64)],
                           lambda o: (o[0].reshape(k_boot, 2), o[1].reshape(k_boot, 13), o[2])),
    "calibrate": ((), lambda n: [out(2, F64), out(1, F64), out(5, I64)], lambda o: (o[0][0], o[0][1], o[1][0], o[2])),
    "calibrate_weighted": ((), lambda n: [out(2, F64), out(1, F64), out(5, I64), out(3, F64)],
                           lambda o: (o[0][0], o[0][1], o[1][0], o[2], o[3])),
    "calibration": ((*SIGMOID, N_BINS), _quality(2), tuple),
    "weighted_calibration": ((*SIGMOID, N_BINS), _wquality(2), tuple),
    "calibrate_isotonic": ((), lambda n: [out(1, I64), out(n, F64), out(n, F64), out(n, I64), out(n, I64), out(5, I64)],
                           _iso_fit),
    "calibrate_isotonic_weighted": ((), lambda n: [out(1, I64), out(n, F64), out(n, F64), out(n, F64), out(n, F64),
                                                   out(5, I64), out(2, F64)], lambda o: (*_iso_fit(o), o[6])),
    "isotonic_calibration": ((*MAP, N_BINS), _quality(3), tuple),
    "weighted_isotonic_calibration": ((*MAP, N_BINS), _wquality(3), tuple),
}


def _camel(s):
    return "".join(p.capitalize() for p in s.split("_"))


def forms(family):
    """[(form, native, NativeCtx method)] of one family"""
    if family.startswith("calibrate"):
        base, rest = "calibrate", _camel(family[len("calibrate"):].lstrip("_"))
        return [("range", base + rest, family), ("drawn", base + rest + "Sampled", family + "_sampled"),
                ("list", base + rest + "Samples", family + "_samples")]
    c = _camel(family)
    return [("range", "eval" + c, "eval_" + family), ("drawn", "evalSampled" + c, "eval_sampled_" + family),
            ("list", "evalSamples" + c, "eval_samples_" + family)]


IDS = np.random.default_rng(5).integers(0, N_ROWS, size=N).astype(np.int32)
ROWS = {"range": (7, 7 + N), "drawn": (7, N_ROWS, KEY - (1 << 64), 5, 5 + N), "list": (IDS,)}


def ctx_call(fn, *args, **kw):
    """(0, result) or (error code, None) of one NativeCtx call"""
    from distributed_sgd_b200.native import DsgdError
    try:
        return 0, fn(*args, **kw)
    except DsgdError as e:
        return e.code, None


@pytest.fixture(scope="module")
def setup(tmp_path_factory):
    from distributed_sgd_b200.native import NativeCtx
    from distributed_sgd_b200.utils import synthetic_rcv1
    data = synthetic_rcv1(n_rows=N_ROWS, seed=23)
    shim = Shim(str(tmp_path_factory.mktemp("jni") / "libdsgd_jni_test.so"))
    rng = np.random.default_rng(23)
    ctxs = {}
    for kind, kw in (("svm", {}), ("logistic_icpt", {"logistic": True, "intercept": True}), ("async", {"is_async": True})):
        c = NativeCtx(0, data.dim, LAM, **kw)
        c.load_csr(data.row_ptr, data.col, data.val, data.label)
        c.compute_dim_sparsity(N_ROWS)
        w = np.where(rng.random(c.wdim) < 0.6, rng.standard_normal(c.wdim) * 0.1, 0.0)
        c.set_weights(w)
        ctxs[kind] = (c, w)
    yield shim, ctxs, data
    for c, _ in ctxs.values():
        c.close()


def _maps_of_libdsgd():
    files = set()
    for line in open("/proc/self/maps"):
        f = line.split()
        if len(f) >= 6 and os.path.basename(f[5]) == "libdsgd.so":
            files.add((f[3], f[4]))
    return files


def test_one_library_copy(setup):
    assert len(_maps_of_libdsgd()) == 1


@pytest.mark.parametrize("kind", ["svm", "logistic_icpt"])
def test_outputs_match_native_ctx(setup, kind):
    shim, ctxs, data = setup
    ctx, w = ctxs[kind]
    h, checked = ctx._h.value, 0
    for family, (tail, outs, to_ctx) in FAMILIES.items():
        for form, jname, method in forms(family):
            rows = ROWS[form]
            o = outs(N)
            rc = shim(jname, h, w, *rows, *tail, *o)
            code, want = ctx_call(getattr(ctx, method), *rows, *tail, w=w)
            assert rc == code, (kind, jname, rc, code)
            if code == 0:
                assert bits(to_ctx(o)) == bits(want), (kind, jname)
            checked += 1
    assert checked == 51
    # the list-only requests, eval, and the weight readers
    for jname, method in (("forward", "forward"), ("margins", "margins"), ("probabilities", "probabilities")):
        o = out(N, F64)
        code, want = ctx_call(getattr(ctx, method), IDS, w)
        assert shim(jname, h, w, IDS, o) == code, jname
        if code == 0:
            assert bits(o) == bits(want), jname
    o = out(N, F64)
    assert shim("calibratedProbabilities", h, w, IDS, *SIGMOID, o) == 0
    assert bits(o) == bits(ctx.calibrated_probabilities(IDS, *SIGMOID, w=w))
    o = out(N, F64)
    assert shim("isotonicProbabilities", h, w, IDS, *MAP, o) == 0
    assert bits(o) == bits(ctx.isotonic_probabilities(IDS, *MAP, w=w))
    g = out(ctx.wdim, F64)
    assert shim("gradient", h, w, IDS, g) == 0
    g_ref = ctx.gradient(IDS, w)
    if ctx.logistic:
        np.testing.assert_allclose(g, g_ref, rtol=1e-12, atol=1e-18)
    else:
        assert bits(g) == bits(g_ref)
    o = out(2, F64)
    assert shim("eval", h, w, 7, 7 + N, o) == 0 and bits(tuple(o)) == bits(ctx.eval(7, 7 + N, w))
    o = out(ctx.wdim, F64)
    assert shim("getWeights", h, o) == 0 and bits(o) == bits(ctx.get_weights())
    l1, nnz = out(1, F64), out(1, I64)
    assert shim("weightsL1", h, w, l1, nnz) == 0 and bits((l1[0], nnz[0])) == bits(ctx.weights_l1(w))
    o = out(ctx.dim, F64)
    assert shim("computeDimSparsity", h, N_ROWS, o) == 0 and bits(o) == bits(ctx.compute_dim_sparsity(N_ROWS))
    assert shim.region_errors() == 0


def _short_cases(ctx, w, data):
    """(native, arguments) with one array of the wrong length, every other argument valid"""
    h, wd, d = ctx._h.value, ctx.wdim, ctx.dim
    cases = [("setWeights", (h, w[:-1])), ("setWeights", (h, np.append(w, 0.0))), ("getWeights", (h, out(wd - 1, F64))),
             ("gradient", (h, w, IDS, out(wd - 1, F64))), ("averageWeights", (h, out(wd - 1, F64), None)),
             ("setDimSparsity", (h, np.ones(d - 1))), ("computeDimSparsity", (h, N_ROWS, out(d - 1, F64))),
             ("forward", (h, w, IDS, out(N - 1, F64))), ("margins", (h, w, IDS, out(N - 1, F64))),
             ("probabilities", (h, w, IDS, out(N - 1, F64))),
             ("calibratedProbabilities", (h, w, IDS, *SIGMOID, out(N - 1, F64))),
             ("isotonicProbabilities", (h, w, IDS, *MAP, out(N - 1, F64))),
             ("loadCsr", (h, data.row_ptr, data.col, data.val, data.label[:-1])),
             ("loadCsr", (h, data.row_ptr, data.col, data.val[:-1], data.label))]
    for bad in (w[:-1], np.append(w, 0.0)):
        cases += [("forward", (h, bad, IDS, out(N, F64))), ("gradient", (h, bad, IDS, out(wd, F64))),
                  ("eval", (h, bad, 7, 7 + N, out(2, F64))), ("weightsL1", (h, bad, out(1, F64), out(1, I64)))]
        for family, (tail, outs, _) in FAMILIES.items():
            cases += [(jname, (h, bad, *ROWS[form], *tail, *outs(N))) for form, jname, _ in forms(family)]
    return cases


@pytest.mark.parametrize("kind", ["svm", "logistic_icpt"])
def test_wrong_lengths_are_refused(setup, kind):
    from distributed_sgd_b200.native import ERR_INVALID
    shim, ctxs, data = setup
    ctx, w = ctxs[kind]
    cases = _short_cases(ctx, w, data)
    assert len(cases) == 14 + 2 * (4 + 51)
    for name, args in cases:
        before, outs = ctx.launch_count(), [a.copy() for a in args if isinstance(a, np.ndarray)]
        assert shim(name, *args) == ERR_INVALID, (kind, name)
        assert ctx.launch_count() == before, (kind, name)
        assert all(np.array_equal(a.view(np.uint8), b.view(np.uint8))
                   for a, b in zip([a for a in args if isinstance(a, np.ndarray)], outs)), (kind, name)
    assert ctx.n_rows == N_ROWS and bits(ctx.get_weights()) == bits(w)      # the refusals changed nothing
    assert shim.region_errors() == 0


def test_async_arrays(setup):
    from distributed_sgd_b200.native import ERR_INVALID
    shim, ctxs, _ = setup
    ctx, w = ctxs["async"]
    h, d = ctx._h.value, ctx.dim
    for name, args in (("asyncHostMaster", (h, np.zeros(d - 1))), ("asyncHostMaster", (h, np.zeros(d + 1))),
                       ("startAsync", (h, np.zeros(d - 1), IDS, 8, 0.1, 1, 16, 1)),
                       ("startAsync", (h, np.zeros(d + 1), IDS, 8, 0.1, 1, 16, 1)),
                       ("asyncMasterWeights", (h, out(d - 1, F64))), ("asyncOutboxRead", (h, out(d - 1, F64)))):
        before = ctx.launch_count()
        assert shim(name, *args) == ERR_INVALID, name
        assert ctx.launch_count() == before and not ctx.async_running(), name
    assert shim("asyncHostMaster", h, w) == 0
    o = out(d, F64)
    assert shim("asyncMasterWeights", h, o) == 0 and bits(o) == bits(ctx.async_master_weights())
    ctx.async_outbox_enable()
    o = out(d, F64)
    assert shim("asyncOutboxRead", h, o) == 0 and bits(o) == bits(ctx.async_outbox_read())
    assert shim.region_errors() == 0


def test_get_weights_from_several_threads(setup):
    """getWeights is one of the calls the header lets run while the async loop runs, from several threads at once: its
    weight-length check reads dsgd_info under the shim's lock, so concurrent calls all give the resident weights."""
    from concurrent.futures import ThreadPoolExecutor
    shim, ctxs, _ = setup
    ctx, _ = ctxs["async"]
    h, want = ctx._h.value, bits(ctx.get_weights())

    def reads(_):
        got = []
        for _ in range(50):
            o = out(ctx.wdim, F64)
            got.append((shim("getWeights", h, o), bits(o)))
        return got

    with ThreadPoolExecutor(8) as pool:
        results = [r for rs in pool.map(reads, range(8)) for r in rs]
    assert len(results) == 400 and all(r == (0, want) for r in results)
    assert shim.region_errors() == 0
