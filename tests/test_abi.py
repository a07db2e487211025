"""The C-ABI library loads and exports every symbol include/gslam_b200.h declares (no compute calls: CPU-safe)."""
import ctypes
import os
import re

import pytest

from gslam_b200 import capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_symbols():
    src = open(os.path.join(ROOT, "include", "gslam_b200.h")).read()
    return sorted(set(re.findall(r"GB_API\s+[\w\s\*]+?\b(gb_\w+)\s*\(", src)))


def test_header_and_binding_agree():
    assert header_symbols() == sorted(capi.EXPORTED_SYMBOLS)


def test_library_exports_every_declared_symbol():
    L = ctypes.CDLL(capi.LIB_PATH)
    for name in header_symbols():
        assert hasattr(L, name), name


def test_version_and_struct_sizes():
    L = capi.lib()
    assert L.gb_version() == 100
    assert ctypes.sizeof(capi.OrbCfg) == 36
    assert capi.KP_DTYPE.itemsize == 28
    o = capi.BaOptions(); L.gb_ba_options_default(ctypes.byref(o))
    # GSLAM::OptimzeConfig defaults (Optimizer.h:174-182)
    assert o.projection == 0 and o.huber_delta == 0.01 and o.max_iterations == 500 and o.verbose == 0
    c = capi.OrbCfg(); L.gb_orb_cfg_default(ctypes.byref(c))
    assert (c.nfeatures, c.nlevels, c.edge_threshold, c.first_level, c.wta_k, c.score_type, c.patch_size, c.fast_threshold) == (500, 8, 31, 0, 2, 0, 31, 20)
    assert abs(c.scale_factor - 1.2) < 1e-6


def test_no_device_fails_loudly():
    """Without a GPU the product refuses to run (no CPU fallback)."""
    L = capi.lib()
    n = ctypes.c_int(-1)
    rc = L.gb_device_count(ctypes.byref(n))
    if rc == 0 and n.value > 0:
        return  # GPU box
    h = ctypes.c_void_p()
    assert L.gb_ctx_create(0, ctypes.byref(h)) == capi.GB_ERR_NODEVICE
    assert h.value is None
    assert len(L.gb_last_error(None)) > 0


def test_product_never_imports_oracle():
    pkg = os.path.join(ROOT, "gslam_b200")
    for dp, _, fs in os.walk(pkg):
        for f in fs:
            if f.endswith((".py", ".cu", ".cuh", ".cpp", ".h")):
                s = open(os.path.join(dp, f), errors="ignore").read()
                assert "import oracle" not in s and "from oracle" not in s and "liboracle" not in s and "orc_" not in s, f


def test_estimator_plugin_exports_the_reference_factory():
    """libgslam_estimator.so is what GSLAM::Estimator::create() dlopens (Estimator.h:175-191): the factory symbol must be there
    and constructing the estimator must not need a device (the context is created lazily, on the first findPnP)."""
    import ctypes
    import oracle
    path = os.path.join(oracle.PLUGIN_DIR, "libgslam_estimator.so")
    if not os.path.exists(path):
        pytest.skip("oracle/_ref/plugins not built (they need the headers of a GSLAM checkout at build time)")
    L = ctypes.CDLL(path)
    L.createEstimatorInstance.restype = ctypes.c_void_p
    assert L.createEstimatorInstance()


def test_header_is_plain_c_and_cpp():
    """include/gslam_b200.h is the boundary other hosts bind (cgo / JNI / ctypes): it must parse as C99 and as C++11 on its own."""
    import shutil
    import subprocess
    import tempfile
    hdr = os.path.join(ROOT, "include", "gslam_b200.h")
    with tempfile.TemporaryDirectory() as d:
        for cc, std, ext in (("gcc", "-std=c99", "c"), ("g++", "-std=c++11", "cpp")):
            if not shutil.which(cc):
                pytest.skip(f"{cc} not available")
            src = os.path.join(d, f"probe.{ext}")
            with open(src, "w") as f:
                f.write('#include "%s"\nint probe(void) { gb_ba_problem p; gb_pose_edges e; gb_orb_cfg c; gb_keypoint k; (void)p; (void)e; (void)c; '
                        '(void)k; return (int)sizeof(gb_keypoint) == 28 ? GB_OK : GB_ERR_INVALID; }\n' % hdr)
            r = subprocess.run([cc, std, "-Wall", "-Werror", "-pedantic", "-fsyntax-only", src], capture_output=True, text=True)
            assert r.returncode == 0, r.stderr
