"""No-GPU checks of the boundary: libevk.so loads, exports every symbol include/evk.h declares,
reports its version, and the host-side argument logic behaves."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    src = open(os.path.join(ROOT, "include", "evk.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(evk_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    from event_utils_b200 import _lib
    L = _lib.load()
    names = declared_symbols()
    assert len(names) >= 25
    for n in names:
        assert hasattr(L, n), "libevk.so does not export %s" % n
    assert L.evk_version() == 100
    assert isinstance(L.evk_last_error(), bytes)


def declared_prototypes():
    """name -> list of parameter type strings, parsed from include/evk.h"""
    src = open(os.path.join(ROOT, "include", "evk.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    protos = {}
    for m in re.finditer(r"\b(?:int|size_t|uint64_t|const char \*|void)\s*\*?\s*(evk_[a-z0-9_]+)\s*\(([^;{]*?)\)\s*;", src, flags=re.S):
        params = [p.strip() for p in m.group(2).replace("\n", " ").split(",")]
        protos[m.group(1)] = [] if params in ([""], ["void"]) else params
    return protos


def test_ctypes_declarations_match_the_header():
    """every prototype of include/evk.h against the argtypes event_utils_b200/_lib.py binds: same number of
    parameters, pointers bound as pointers, 64-bit integers as 64-bit, floats / doubles as such"""
    from event_utils_b200 import _lib
    L = _lib.load()
    protos = declared_prototypes()
    assert len(protos) == len(declared_symbols()) and "evk_voxel_f32" in protos and "evk_voxel_fold_allreduce_f32" in protos

    def kind(c_type):
        c = c_type.replace("const ", "").strip()
        c = re.sub(r"\b[A-Za-z_][A-Za-z0-9_]*$", "", c).strip() if not c.endswith("*") else c   # drop the parameter name
        if "*" in c_type:
            return "ptr"
        for key, val in (("uint64_t", "size"), ("int64_t", "i64"), ("size_t", "size"), ("unsigned", "u32"), ("double", "f64"), ("float", "f32"), ("int", "i32")):
            if re.search(r"\b%s\b" % key, c_type):
                return val
        raise AssertionError("unparsed parameter type %r" % c_type)

    bound = {ctypes.c_void_p: "ptr", ctypes.c_char_p: "ptr", ctypes.c_int64: "i64", ctypes.c_longlong: "i64", ctypes.c_size_t: "size",
             ctypes.c_uint: "u32", ctypes.c_double: "f64", ctypes.c_float: "f32", ctypes.c_int: "i32"}
    checked = 0
    for name, params in protos.items():
        fn = getattr(L, name)
        if fn.argtypes is None:
            continue                      # not bound by the python layer (e.g. used from C only)
        assert len(fn.argtypes) == len(params), "%s: header has %d parameters, _lib.py binds %d" % (name, len(params), len(fn.argtypes))
        for i, (c_type, at) in enumerate(zip(params, fn.argtypes)):
            got = "ptr" if (isinstance(at, type) and issubclass(at, ctypes._Pointer)) else bound.get(at)
            want = kind(c_type)
            if want == "size" and got == "i64":
                got = "size"
            assert got == want, "%s parameter %d (%s): bound as %s" % (name, i, c_type, at)
        checked += 1
    assert checked >= 30


def test_workspace_queries_need_no_gpu():
    from event_utils_b200 import _lib
    L = _lib.load()
    VR = _lib.VARIANT_VECTOR_RED
    def quads(nbytes):                     # the quad workspace, 256-byte aligned, + 256 bytes for the launch-level contention verdict
        return (nbytes + 255) // 256 * 256 + 256
    assert L.evk_voxel_workspace_bytes(5, 480, 640, VR) == quads(480 * 640 * 2 * 16)   # two quads per pixel
    assert L.evk_voxel_workspace_bytes(1, 10, 10, VR) == quads(10 * 10 * 16)
    assert L.evk_voxel_workspace_bytes(4, 10, 10, VR) == quads(10 * 10 * 16)
    assert L.evk_voxel_workspace_bytes(8, 10, 10, VR) == quads(10 * 10 * 3 * 16)
    # AUTO / ROUTED also cover the routed kernel's rings (one 128 KB ring per SM + its counters)
    assert L.evk_voxel_workspace_bytes(5, 480, 640, 0) >= 480 * 640 * 2 * 16
    assert 132 * 16384 * 8 <= L.evk_voxel_workspace_bytes(5, 480, 640, _lib.VARIANT_ROUTED) <= L.evk_voxel_workspace_bytes(5, 480, 640, 0)
    assert L.evk_image_workspace_bytes(181, 241, _lib.BILINEAR) == 181 * 241 * 16
    assert L.evk_voxel_workspace_bytes(5, 481, 641, _lib.BILINEAR) == 5 * 481 * 641 * 16
    assert L.evk_image_workspace_bytes(181, 241, 0) == 0
    assert L.evk_cmax_workspace_bytes(180, 240) >= 8 * 181 * 241 * 16


def test_compute_fails_loudly_without_gpu():
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from event_utils_b200 import _lib
    from event_utils_b200.representations.voxel_grid import events_to_voxel_torch
    with pytest.raises(_lib.EvkError):
        _lib.lib()
    x = torch.zeros(4)
    with pytest.raises(_lib.EvkError):
        events_to_voxel_torch(x, x, torch.arange(4.0), x, 3)


def test_host_side_argument_logic():
    from event_utils_b200.representations import _events as E
    from event_utils_b200.representations.image import _canvas_and_clip
    from event_utils_b200.representations.voxel_grid import events_to_voxel_torch
    # image.py:64-67, 73-74
    assert _canvas_and_clip((180, 240), None, True) == ((180, 240), 239.0, 179.0)
    assert _canvas_and_clip((180, 240), None, False) == ((180, 240), 240.0, 180.0)
    assert _canvas_and_clip((180, 240), 'bilinear', True) == ((181, 241), 240.0, 180.0)
    assert _canvas_and_clip((180, 240), 'bilinear', False) == ((180, 240), 239.0, 179.0)
    # AoS detection
    ev = torch.arange(40, dtype=torch.float32).reshape(10, 4)
    assert E.aos_base(ev[:, 0], ev[:, 1], ev[:, 2], ev[:, 3]) is not None
    assert E.aos_base(ev[:, 1], ev[:, 0], ev[:, 2], ev[:, 3]) is None
    assert E.aos_base(ev[:, 0].clone(), ev[:, 1], ev[:, 2], ev[:, 3]) is None
    # reference error conventions that do not need the GPU
    x = torch.zeros(4)
    with pytest.raises(AssertionError):
        events_to_voxel_torch(x, x[:3], x, x, 3)
    with pytest.raises(NotImplementedError):
        events_to_voxel_torch(x, x, x, x, 3, temporal_bilinear=False)
    with pytest.raises(IndexError):
        events_to_voxel_torch(x[:0], x[:0], x[:0], x[:0], 3)


def test_bounds_mask_known_answer():
    from event_utils_b200.util.event_util import events_bounds_mask
    m = events_bounds_mask(np.array([0, 1e-9, 240, 240.1]), np.array([5.0, 5, 5, 5]), 0, 240, 0, 180)
    assert m.tolist() == [0.0, 1.0, 1.0, 0.0]


def test_argument_errors_are_reported_without_touching_the_gpu():
    """Bad arguments come back as EVK_E_ARG / EVK_E_WORKSPACE with a message, before any CUDA call."""
    from event_utils_b200 import _lib
    L = _lib.load()
    one = ctypes.c_void_p(16)   # a non-null, aligned, never dereferenced pointer
    assert L.evk_voxel_f32(None, one, one, one, 10, 0.0, 1.0, 5, 4, 4, 0, one, None, 0, None, None) == -1
    assert b"null event array" in L.evk_last_error()
    assert L.evk_voxel_f32(one, one, one, one, -1, 0.0, 1.0, 5, 4, 4, 0, one, None, 0, None, None) == -1
    assert L.evk_voxel_f32(one, one, one, one, 10, 0.0, 1.0, 0, 4, 4, 0, one, None, 0, None, None) == -1
    # vector-red variant without a workspace
    assert L.evk_voxel_f32(one, one, one, one, 10, 0.0, 1.0, 5, 4, 4, _lib.VARIANT_VECTOR_RED, one, None, 0, None, None) == -3
    assert b"workspace" in L.evk_last_error()
    assert L.evk_image_f32(one, one, one, 10, 1, 1, 0.0, 0.0, _lib.BILINEAR, 0.0, one, None, 0, None, None) == -1
    assert L.evk_image_f32(one, one, None, 10, 4, 4, 0.0, 0.0, 0, 0.0, one, None, 0, None, None) == -1
    assert L.evk_cmax_linvel_variance_f64(one, one, one, one, 10, 1.0, 0.0, 0.0, 0.0, 180, 240, 180, 240, 1.0, 0,
                                          one, None, None, None, 0, None) == -1
    assert L.evk_timestamp_image_f32(one, one, one, one, 10, 0.0, 1.0, 4, 4, 3.0, 3.0, 0, one, one, None, 0, None, None) == -3
    assert L.evk_warp_flow_f32(one, one, one, 10, None, 4, 4, 0.0, one, one, None, 0, None) == -1
    assert L.evk_voxel_windows_f32(one, one, one, one, None, 3, 0, 5, 4, 4, 0, one, None, None) == -1
    assert L.evk_voxel_negpos_f32(one, one, one, one, 10, 0.0, 1.0, 5, 4, 4, _lib.BILINEAR, one, None, 0, None, None) == -5


def test_header_is_plain_c99(tmp_path):
    """include/evk.h compiles as C99 and as C++ without CUDA or torch headers, and names every entry point"""
    import shutil
    import subprocess
    if shutil.which("gcc") is None:
        pytest.skip("no gcc")
    src = tmp_path / "use_evk.c"
    uses = "\n".join("    (void)&%s;" % n for n in declared_symbols())
    src.write_text('#include "evk.h"\nint main(void)\n{\n%s\n    return 0;\n}\n' % uses)
    inc = os.path.join(ROOT, "include")
    for cmd in (["gcc", "-std=c99", "-Wall", "-Werror", "-fsyntax-only", "-I", inc, str(src)],
                ["g++", "-x", "c++", "-Wall", "-Werror", "-fsyntax-only", "-I", inc, str(src)]):
        if shutil.which(cmd[0]) is None:
            continue
        r = subprocess.run(cmd, capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
