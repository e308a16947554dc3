"""The C-ABI shared library: it loads without a GPU, exports every symbol include/michigan_b200.h
declares, the ctypes signatures cover the header, and argument errors are reported through the
status-code / mg_last_error() convention (no compute calls here)."""
import ctypes as C
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "michigan_b200.h")


def declared_functions():
    src = open(HEADER).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(mg_[a-z0-9_]+)\s*\(", src)))


def test_header_declares_a_plain_c_abi():
    src = open(HEADER).read()
    assert 'extern "C"' in src
    assert "torch" not in re.sub(r"/\*.*?\*/", "", src, flags=re.S).lower()
    assert len(declared_functions()) >= 25


def test_library_exports_every_declared_symbol():
    from michigan_b200 import _lib
    lib = C.CDLL(_lib.LIB_PATH)
    for name in declared_functions():
        assert hasattr(lib, name), "symbol %s declared in the header but not exported" % name


def test_ctypes_signatures_and_abi_version_match_the_header():
    from michigan_b200 import _lib
    assert sorted(_lib.SIGNATURES) == declared_functions()
    lib = _lib.load()
    assert lib.mg_version() == 3
    assert lib.mg_launch_count() >= 0


def test_struct_layouts_match_the_header():
    """Field order/count of the ctypes structures against the C typedefs."""
    from michigan_b200 import _lib
    src = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    for cname, st in (("mg_igemm_args", _lib.IgemmArgs), ("mg_thin_args", _lib.ThinArgs)):
        body = re.search(r"typedef struct %s \{(.*?)\} %s;" % (cname, cname), src, flags=re.S).group(1)
        fields = []
        for decl in body.split(";"):
            decl = decl.strip()
            if not decl:
                continue
            names = re.sub(r"^(const\s+)?(float\*|void\*|int32_t|float)\s*", "", decl)
            fields += [n.strip().lstrip("*") for n in names.split(",")]
        got = [("in" if f[0] == "inp" else f[0]) for f in st._fields_]
        assert got == fields, (cname, got, fields)


def test_argument_errors_use_status_codes_without_touching_the_gpu():
    from michigan_b200 import _lib
    lib = _lib.load()
    assert lib.mg_pack_weight(None, None, 1, 1, 1, 1, None, 0, None) < 0
    assert b"null" in lib.mg_last_error()
    a = _lib.IgemmArgs()
    assert lib.mg_conv_igemm(C.byref(a), None) < 0
    a.inp = a.wpack = a.out = 4096
    a.Cin = 48
    assert lib.mg_conv_igemm(C.byref(a), None) == -2 and b"multiple of 32" in lib.mg_last_error()
    with pytest.raises(_lib.MichiganNativeError):
        _lib.check(-2, "demo")


def test_ops_refuse_cpu_tensors():
    """There is no CPU fallback: host tensors are rejected loudly."""
    import torch
    from michigan_b200 import _lib, ops
    with pytest.raises(_lib.MichiganNativeError):
        ops.bn_sums(torch.zeros(1, 4, 4, 8))
    with pytest.raises(_lib.MichiganNativeError):
        ops.pack_weight(torch.zeros(32, 32, 3, 3))


def test_header_knobs_exist_and_retired_knobs_are_rejected():
    """Every schedule knob the header documents is known to mg_get_tuning / mg_set_tuning (host-only calls); unknown names fail,
    and so do the retired names of knobs that had no effect on sm_90a."""
    import re
    from michigan_b200 import _lib
    lib = _lib.load()
    text = open(os.path.join(ROOT, "include", "michigan_b200.h")).read()
    names = sorted(set(re.findall(r'"(MG_[A-Z0-9_]+)"', text)))
    assert {"MG_GROUP3", "MG_SEG_TMA", "MG_EPI_REG", "MG_MERGE"} <= set(names)
    for n in names:
        v = lib.mg_get_tuning(n.encode())
        assert v > -(1 << 30), n
        assert lib.mg_set_tuning(n.encode(), v) == 0, n
    assert lib.mg_set_tuning(b"MG_NO_SUCH_KNOB", 1) < 0
    for n in ("MG_DUAL", "MG_WGRAD_DUAL", "MG_WGRAD_HALO", "MG_EPI_TMA", "MG_EPI_EARLY"):
        assert lib.mg_set_tuning(n.encode(), 1) == -2, n
