"""CPU tests (no GPU): every kernel of libsslpl_b200 is launched and counted in one place, launch() in csrc/common.cuh, and the
handle plumbing of csrc/common.cuh's StreamHandle is not written out again in a .cu file."""
import glob
import os
import re

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "structure-slam-pointline_b200", "csrc")


def _source(path):
    return re.sub(r"//[^\n]*|/\*.*?\*/", "", open(path).read(), flags=re.S)


def _cu_files():
    files = sorted(glob.glob(os.path.join(CSRC, "*.cu")))
    assert len(files) >= 5
    return {os.path.basename(f): _source(f) for f in files}


def test_every_kernel_launch_is_in_launch():
    common = _source(os.path.join(CSRC, "common.cuh"))
    assert common.count("<<<") == 1
    body = re.search(r"\bvoid launch\(StreamHandle\* h,[^{]*\{([^}]*)\}", common).group(1)
    assert "<<<" in body and "h->launches++" in body
    for name, src in _cu_files().items():
        assert "<<<" not in src, name


def test_no_cu_file_writes_the_launch_count():
    for name, src in _cu_files().items():
        assert not re.search(r"launches\s*(\+\+|[-+]?=(?!=))|\+\+\s*\w+->launches", src), name


def test_no_cu_file_redefines_the_handle_helpers():
    for name, src in _cu_files().items():
        assert not re.search(r"\b(?:void|int)\s+(\w*mark|check_device_err|ensure_scratch|first_use)\s*\(", src), name
