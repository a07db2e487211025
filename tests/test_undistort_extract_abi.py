"""The device-resident undistortion calls are declared, exported and bound with the documented prototypes (no device needed)."""
import ctypes as C
import os
import re

from gslam_b200 import capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
VP, I = C.c_void_p, C.c_int
# C parameter type -> ctypes type, in the order of the declarations in include/gslam_b200.h
DOCUMENTED = {
    "gb_remap_apply_to": ("gb_ctx*, gb_remap*, const uint8_t*, int, int, int, uint8_t*, int", [VP, VP, VP, I, I, I, VP, I]),
    "gb_orb_extract_undistorted_to": ("gb_ctx*, gb_remap*, const uint8_t*, int, int, int, int, const gb_orb_cfg*, gb_features*",
                                      [VP, VP, VP, I, I, I, I, C.POINTER(capi.OrbCfg), VP]),
    "gb_orb_extract_undistorted": ("gb_ctx*, gb_remap*, const uint8_t*, int, int, const gb_orb_cfg*, gb_keypoint*, uint8_t*, int*",
                                   [VP, VP, VP, I, I, C.POINTER(capi.OrbCfg), VP, VP, C.POINTER(I)]),
}


def test_prototypes_declared_exported_and_bound():
    hdr = open(os.path.join(ROOT, "include", "gslam_b200.h")).read()
    bound = {name: (res, args) for name, res, args in capi._SIGNATURES}
    L = C.CDLL(capi.LIB_PATH)
    for name, (c_types, argtypes) in DOCUMENTED.items():
        m = re.search(r"GB_API\s+int\s+%s\s*\(([^)]*)\)\s*;" % name, hdr)
        assert m, name
        params = [re.sub(r"\s+", " ", p).strip() for p in m.group(1).split(",")]
        declared = ", ".join(re.sub(r"\s*\b\w+$", "", p) for p in params)   # drop the parameter names
        assert declared == c_types, (name, declared)
        assert hasattr(L, name), name
        assert bound[name] == (C.c_int, argtypes), name
    assert capi.lib().gb_version() == 100
