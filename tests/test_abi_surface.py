"""The C-ABI library loads on a machine without a GPU and exports every symbol include/dsgd.h declares; the
ctypes binding covers the same set; without a GPU the library fails loudly (no CPU fallback)."""
import ctypes as C
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    text = open(os.path.join(ROOT, "include", "dsgd.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(dsgd_[a-z0-9_]+)\s*\(", text)))


def test_library_exports_every_declared_symbol():
    from distributed_sgd_b200 import native
    lib = C.CDLL(native.LIB_PATH)
    names = declared_symbols()
    assert len(names) >= 40
    for n in names:
        assert hasattr(lib, n), f"{n} declared in dsgd.h but not exported by libdsgd.so"


def test_ctypes_binding_covers_the_header():
    from distributed_sgd_b200 import native
    assert sorted(native.ABI) == declared_symbols()
    native.lib()                                   # resolves every bound symbol with its argtypes


def declared_parameter_kinds():
    """{name: [kind of each parameter]} of every prototype in include/dsgd.h: ptr, i32, u32, i64, u64 or f64"""
    text = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "dsgd.h")).read(), flags=re.S)
    scalar = {"int": "i32", "int32_t": "i32", "uint32_t": "u32", "int64_t": "i64", "uint64_t": "u64", "double": "f64"}
    out = {}
    for name, params in re.findall(r"^(?:int|const char \*)\s*(dsgd_\w+)\(([^)]*)\);", text, re.M):
        out[name] = ["ptr" if "*" in p or "[" in p else scalar[p.split()[0]] for p in params.split(",")]
    return out


def test_ctypes_argtypes_match_the_header_prototypes():
    """Every ABI entry, the generated row forms included, has its prototype's arity and each parameter's kind."""
    from distributed_sgd_b200 import native
    kind = {C.c_void_p: "ptr", C.c_char_p: "ptr", C.c_int32: "i32", C.c_uint32: "u32", C.c_int64: "i64", C.c_uint64: "u64",
            C.c_double: "f64"}
    declared = declared_parameter_kinds()
    assert sorted(declared) == declared_symbols()
    for name, args in native.ABI.items():
        got = ["ptr" if issubclass(t, C._Pointer) else kind[t] for t in args]
        assert got == declared[name], name


def test_row_methods_name_a_bound_native_ctx_method_for_every_form():
    """Master reaches every form of an evaluation family through native.row_methods: each name is a NativeCtx method, and
    dsgd_<name> is bound."""
    from distributed_sgd_b200 import native
    for family in [*native._ROW_FAMILIES, "eval_topics", "eval_topic_ranking"]:
        methods = native.row_methods(family)
        assert sorted(methods) == ["drawn", "list", "range"], family
        for name in methods.values():
            assert callable(getattr(native.NativeCtx, name, None)) and "dsgd_" + name in native.ABI, name


def row_form_entry_points():
    """dsgd_eval and the range, drawn-sample and id-list forms of the fifteen evaluation families"""
    evals = ["counts", "sums", "class", "weighted", "metrics", "curve", "weighted_curve", "calibration",
             "weighted_calibration", "isotonic_calibration", "weighted_isotonic_calibration"]
    fits = ["calibrate", "calibrate_weighted", "calibrate_isotonic", "calibrate_isotonic_weighted"]
    return (["dsgd_eval"] + [f"dsgd_eval{form}_{e}" for e in evals for form in ("", "_sampled", "_samples")]
            + [f"dsgd_{f}{form}" for f in fits for form in ("", "_sampled", "_samples")])


def test_row_form_entry_points_refuse_a_null_ctx():
    """Every evaluation entry point returns DSGD_ERR_INVALID for a NULL ctx before it reads any other argument."""
    from distributed_sgd_b200 import native
    names = row_form_entry_points()
    assert len(names) == len(set(names)) == 46 and set(names) <= set(declared_symbols())
    lib = native.lib()
    for n in names:
        fn = getattr(lib, n)
        args = [0.0 if t is C.c_double else 0 if t in (C.c_int32, C.c_int64, C.c_uint64) else None
                for t in fn.argtypes[1:]]
        assert fn(None, *args) == native.ERR_INVALID, n


def test_no_cpu_fallback_without_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    from distributed_sgd_b200 import native
    with pytest.raises(native.DsgdError) as e:
        native.NativeCtx(0, 16, 0.1)
    assert e.value.code == native.ERR_CUDA and "no CPU path" in str(e.value)


def test_product_never_imports_the_oracle():
    """The product path must not route through the checker: no Python import of `oracle`, no C include of it."""
    pkg = os.path.join(ROOT, "distributed_sgd_b200")
    pat_py = re.compile(r"^\s*(from\s+oracle\b|import\s+oracle\b|from\s+\.+oracle\b)", re.M)
    pat_c = re.compile(r'#include\s+["<][^">]*oracle', re.M)
    for d, _, files in os.walk(pkg):
        for f in files:
            path = os.path.join(d, f)
            if f.endswith(".py"):
                assert not pat_py.search(open(path).read()), f"{path} imports the oracle"
            elif f.endswith((".cu", ".cuh", ".c", ".h")):
                assert not pat_c.search(open(path).read()), f"{path} includes the oracle"
    assert "oracle" not in open(os.path.join(pkg, "csrc", "Makefile")).read()


def test_jni_shim_type_checks_and_covers_every_native(tmp_path):
    """distributed_sgd_b200/jni/dsgd_jni.c against include/dsgd.h through a stand-in jni.h (no JDK in the image): it
    compiles warning-free, and it exports exactly one Java_..._<name> per `@native def` of DsgdNative.scala."""
    import re
    import shutil
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else shutil.which("gcc")
    if cc is None:
        pytest.skip("no C compiler")
    obj = str(tmp_path / "dsgd_jni.o")
    subprocess.run([cc, "-std=gnu11", "-Wall", "-Wextra", "-Wno-unused-parameter", "-Werror", "-fPIC", "-DDSGD_HAVE_JNI",
                    "-I" + os.path.join(root, "tests", "jni_mock"), "-I" + os.path.join(root, "include"), "-c",
                    os.path.join(root, "distributed_sgd_b200", "jni", "dsgd_jni.c"), "-o", obj], check=True)
    syms = subprocess.run(["nm", "-g", "--defined-only", obj], check=True, capture_output=True, text=True).stdout
    exported = {m.group(1) for m in re.finditer(r" T Java_epfl_distributed_nativ_DsgdNative_00024_(\w+)", syms)}
    scala = open(os.path.join(root, "distributed_sgd_b200", "jni", "DsgdNative.scala")).read()
    natives = set(re.findall(r"@native def (\w+)\(", scala))
    assert natives and exported == natives
    undefined = subprocess.run(["nm", "-u", obj], check=True, capture_output=True, text=True).stdout
    called = set(re.findall(r"U (dsgd_\w+)", undefined))
    header = open(os.path.join(root, "include", "dsgd.h")).read()
    assert called and all(re.search(r"\b%s\(" % c, header) for c in called)     # only functions the header declares
    # the facade covers the header: everything a JVM Master / Slave needs, including the multi-GPU and async membership
    # calls (core/Master.scala:222-243; core/Slave.scala:159-195).  Left out on purpose: host-side stopwatches and the
    # staged-sample split of the bench harness, developer aids, and dsgd_sync_step (= dsgd_sync_steps with one step).
    not_bound = {"dsgd_last_error", "dsgd_create", "dsgd_destroy",               # bound, but nm lists them too: fine either way
                 "dsgd_info", "dsgd_set_stream", "dsgd_synchronize", "dsgd_timer_start", "dsgd_timer_stop", "dsgd_launch_count",
                 "dsgd_profile_begin", "dsgd_profile_end", "dsgd_set_grid_limit", "dsgd_reserve", "dsgd_debug_timeline", "dsgd_sync_step",
                 "dsgd_stage_samples", "dsgd_sync_steps_staged", "dsgd_read_losses", "dsgd_async_replay", "dsgd_async_elapsed_ms"}
    declared = set(re.findall(r"^(?:int|const char \*)\s*(dsgd_\w+)\(", header, re.M))
    missing = declared - called - not_bound
    assert not missing, f"header functions without a JNI native: {sorted(missing)}"
    # blocking GPU calls must not sit inside a critical region (JNI forbids it; GC stall / deadlock across ranks)
    shim = open(os.path.join(root, "distributed_sgd_b200", "jni", "dsgd_jni.c")).read()
    code = re.sub(r"/\*.*?\*/", "", shim, flags=re.S)
    assert "GetPrimitiveArrayCritical" not in code and "ArrayElements" not in code
