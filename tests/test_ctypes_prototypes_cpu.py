"""CPU tests (no GPU): the Python layer binds every function of include/sslpl.h with the header's prototype, so ctypes converts each
argument to its C parameter type, and every call site passes the header's number of arguments."""
import ast
import ctypes as C
import os
import re
import subprocess
import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG_DIR = os.path.join(ROOT, "structure-slam-pointline_b200")


def _header_arity():
    """{name: number of parameters} of every sslpl_* function, read independently of the package's parser."""
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "sslpl.h")).read(), flags=re.S)
    return {name: 0 if params.strip() == "void" else params.count(",") + 1
            for name, params in re.findall(r"\b(sslpl_[a-z0-9_]+)\s*\(([^)]*)\)", hdr)}


def _exported():
    """The sslpl_* functions the built library exports (its dynamic symbol table), independent of both headers' parsers."""
    so = os.path.join(PKG_DIR, "libsslpl_b200.so")
    out = subprocess.run(["nm", "-D", "--defined-only", so], capture_output=True, text=True, check=True).stdout
    return {line.split()[-1] for line in out.splitlines() if line.split() and line.split()[-1].startswith("sslpl_")}


def test_every_exported_function_has_its_header_prototype(pkg):
    """include/sslpl.h declares exactly the library's exports outside include/sslpl_map.h, and each is bound with its prototype."""
    lib = pkg.lib()
    arity = _header_arity()
    map_fns = {"sslpl_update_map_points_batch_device", "sslpl_update_map_lines_batch_device"}
    assert set(arity) == _exported() - map_fns
    mapped = {C.c_void_p, C.c_int, C.c_float, C.c_double, C.c_size_t, C.c_longlong}
    for name, n in arity.items():
        argtypes = getattr(lib, name).argtypes
        assert argtypes is not None and len(argtypes) == n, (name, argtypes, n)
        assert all(t in mapped for t in argtypes), (name, argtypes)


def test_prototype_spot_checks(pkg):
    lib = pkg.lib()
    assert lib.sslpl_last_error.restype is C.c_char_p and lib.sslpl_last_error.argtypes == []
    for kind in ("orb", "matcher", "line", "frame"):
        assert getattr(lib, f"sslpl_{kind}_launch_count").restype is C.c_longlong
        assert getattr(lib, f"sslpl_{kind}_stream").restype is C.c_void_p
    assert lib.sslpl_frame_orb.restype is C.c_void_p and lib.sslpl_frame_line.restype is C.c_void_p
    for kind in ("orb", "matcher", "line", "frame", "vocab"):
        assert getattr(lib, f"sslpl_{kind}_destroy").restype is None
    for kind in ("orb", "line"):
        assert getattr(lib, f"sslpl_{kind}_extract_batch_device").argtypes[-1] is C.c_size_t
    assert lib.sslpl_frame_set_camera.argtypes == [C.c_void_p, C.c_float, C.c_float, C.c_float, C.c_float, C.c_void_p, C.c_int]
    assert lib.sslpl_frame_stream.argtypes == [C.c_void_p, C.c_int]
    assert lib.sslpl_frame_debug_undistort.argtypes == [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    assert lib.sslpl_predict_scale_table.argtypes == [C.c_float, C.c_int, C.c_void_p]


def test_unmapped_scalar_type_raises(pkg):
    assert pkg._prototypes("long long sslpl_x(const float* a, size_t n);") == {"sslpl_x": (C.c_longlong, [C.c_void_p, C.c_size_t])}
    with pytest.raises(pkg.SslplError, match="unsigned short"):
        pkg._prototypes("int sslpl_x(void* h, unsigned short v);")


def test_call_sites_pass_the_header_arity():
    """ctypes passes extra arguments through even with argtypes set, so count them at every lib().sslpl_*(...) call."""
    arity = _header_arity()
    checked = 0
    for f in ("__init__.py", "batch.py"):
        tree = ast.parse(open(os.path.join(PKG_DIR, f)).read())
        for node in ast.walk(tree):
            if not (isinstance(node, ast.Call) and isinstance(node.func, ast.Attribute) and node.func.attr.startswith("sslpl_")
                    and isinstance(node.func.value, ast.Call) and getattr(node.func.value.func, "id", None) == "lib"):
                continue
            if any(isinstance(a, ast.Starred) for a in node.args):
                continue
            assert not node.keywords and len(node.args) == arity[node.func.attr], (f, node.lineno, node.func.attr)
            checked += 1
    assert checked >= 70                    # the walk does find the call sites


def test_integer_reaches_a_float_parameter_as_its_value(pkg):
    """sslpl_orb_tables_host is host arithmetic only: a Python int scale factor must arrive as the float 2.0."""
    sc, isc, s2, is2 = (np.zeros(8, np.float32) for _ in range(4))
    nf = np.zeros(8, np.int32); um = np.zeros(16, np.int32)
    rc = pkg.lib().sslpl_orb_tables_host(1000, 2, 8, *(a.ctypes.data_as(C.c_void_p) for a in (sc, isc, s2, is2, nf, um)))
    assert rc == 0
    assert np.array_equal(sc, 2.0 ** np.arange(8, dtype=np.float32)) and np.array_equal(s2, sc * sc)
