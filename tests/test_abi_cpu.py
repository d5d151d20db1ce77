"""CPU-side checks of the drop-in boundary: the C-ABI library loads without a GPU, exports every symbol that
include/pfd_b200.h declares, and the ctypes binding declares each one with the header's types (no compute calls are
made here)."""
import ctypes
import os
import re
import types
from ctypes import POINTER, c_char_p, c_float, c_int32, c_int64, c_uint32

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "pfd_b200.h")


def _declared():
    src = open(HEADER).read()
    return sorted(set(re.findall(r"PFD_API\s+[\w\s\*]+?\b(pfd_\w+)\s*\(", src)))


class _StubLib:
    """Stands in for the CDLL: every attribute is a plain object that records argtypes / restype."""

    def __init__(self, lacks=()):
        self._lacks = set(lacks)

    def __getattr__(self, name):
        if name.startswith("_") or name in self._lacks:
            raise AttributeError(name)
        fn = types.SimpleNamespace()
        setattr(self, name, fn)
        return fn


def test_header_declares_entry_points():
    names = _declared()
    assert "pfd_gemm_f16" in names and "pfd_groupnorm_f16" in names and len(names) >= 15


def test_library_exports_every_declared_symbol():
    from pfd_b200 import native
    lib = native.load()
    for name in _declared():
        assert hasattr(lib, name), f"{name} declared in include/pfd_b200.h but not exported"
    assert lib.pfd_version() == 2


def _expected_types(decl):
    """ctypes types of a header declaration 'type name' (or a bare return type), written independently of native."""
    decl = " ".join(decl.replace("*", " * ").split())
    if decl.count("*"):
        head = decl[:decl.rindex("*")].strip()
        if head == "const char":
            return c_char_p
        if head == "const pfd_gemm_desc":
            return "gemm_desc"
        return "ptr"
    base = decl.split()[0]
    return {"int": c_int32, "int32_t": c_int32, "uint32_t": c_uint32, "int64_t": c_int64, "float": c_float}[base]


def test_python_binding_lists_match_header():
    """Every prototype gets argtypes of the header's length and the header's type at each position, and its restype."""
    from pfd_b200 import native
    assert sorted(native.EXPORTS) == _declared()
    lib = native._declare(_StubLib())
    src = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    protos = re.findall(r"PFD_API\s+([\w\s\*]+?)\s*\b(pfd_\w+)\s*\(([^)]*)\)", src)
    assert len(protos) == len(native.EXPORTS)
    resolve = {"ptr": native.DevicePtr, "gemm_desc": POINTER(native.GemmDesc)}
    for ret, name, params in protos:
        fn = getattr(lib, name)
        params = [p.strip() for p in params.split(",") if p.strip() not in ("", "void")]
        assert len(fn.argtypes) == len(params), name
        for i, (decl, got) in enumerate(zip(params, fn.argtypes)):
            want = _expected_types(re.sub(r"\w+$", "", decl))
            assert got is resolve.get(want, want), f"{name} argument {i} ({decl}): {got}"
        want = _expected_types(ret)
        assert fn.restype is resolve.get(want, want), f"{name} returns {ret}: {fn.restype}"
    # a few signatures written out by hand
    P = native.DevicePtr
    assert lib.pfd_axpby_f16.argtypes == [P, c_float, P, c_float, c_int64, P, P]
    assert lib.pfd_randn_f16.argtypes == [P, c_int32, c_int64, P, c_uint32, c_int32, P, c_float, P]
    assert lib.pfd_hed_fuse_f32.argtypes == [P, P, P, c_int32, c_int32, c_int32, c_int32, c_float, P, P]
    assert lib.pfd_set_option.argtypes == [c_char_p, c_int32] and lib.pfd_set_option.restype is c_int32
    assert lib.pfd_gemm_f16.argtypes == [POINTER(native.GemmDesc)]
    assert lib.pfd_version.argtypes == [] and lib.pfd_version.restype is c_int32
    assert lib.pfd_canny_workspace_bytes.argtypes == [c_int32] * 3
    assert lib.pfd_canny_workspace_bytes.restype is c_int64
    assert lib.pfd_launch_count.restype is c_int64
    assert lib.pfd_last_error.restype is c_char_p


def test_unknown_header_type_is_rejected(tmp_path, monkeypatch):
    from pfd_b200 import native
    header = tmp_path / "pfd_b200.h"
    header.write_text("PFD_API int pfd_version(void);\nPFD_API int pfd_axpby_f16(const void* a, double sa);\n")
    monkeypatch.setattr(native, "HEADER", str(header))
    monkeypatch.setattr(native, "_lib", None)
    with pytest.raises(RuntimeError, match=r"pfd_axpby_f16.*'double'"):
        native.load()


def test_missing_symbol_is_named():
    from pfd_b200 import native
    with pytest.raises(RuntimeError, match="pfd_softmax_f16, pfd_mlsd_head_f32"):
        native._declare(_StubLib(lacks=("pfd_softmax_f16", "pfd_mlsd_head_f32")))


def test_pointer_arguments_take_tensors_and_refuse_host_tensors():
    """A CPU tensor in a pointer argument raises ctypes.ArgumentError before any C code runs; ints, None, ctypes arrays
    and byref pass through as c_void_p does."""
    from pfd_b200 import native
    lib = native.load()
    n0 = lib.pfd_launch_count()
    a = torch.zeros(8, dtype=torch.float16)
    with pytest.raises(ctypes.ArgumentError, match="argument 1: .*CUDA"):
        lib.pfd_axpby_f16(a, 1.0, None, 0.0, 8, a, None)
    with pytest.raises(ctypes.ArgumentError, match="argument 6: .*CUDA"):
        lib.pfd_axpby_f16(0, 1.0, None, 0.0, 8, a, None)
    assert lib.pfd_launch_count() == n0
    strlen = ctypes.CDLL(None).strlen
    strlen.argtypes, strlen.restype = [native.DevicePtr], ctypes.c_size_t
    buf = ctypes.create_string_buffer(b"abcd")
    assert strlen(buf) == strlen(ctypes.byref(buf)) == strlen(ctypes.addressof(buf)) == 4
    assert native.DevicePtr.from_param(None) is None


def test_header_constants_match_python_mirrors():
    from pfd_b200 import native
    src = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    defines = dict(re.findall(r"^#define[ \t]+(PFD_\w+)[ \t]+(\S.*?)\s*$", src, flags=re.M))
    names = [n for n in defines if hasattr(native, n)]
    assert sorted(names) == sorted(["PFD_MAX_SEG", "PFD_KSAMPLER_NCOEF", "PFD_HED_MAX_SIDES", "PFD_PIDINET_SIDE_PARAMS",
                                    "PFD_MLSD_TOPK", "PFD_OPENPOSE_MAX_PEAKS", "PFD_OPENPOSE_MAX_PERSONS"])
    values = {}
    for n in names:
        values[n] = eval(defines[n], {}, values)           # the header's own expression, over the defines before it
        assert getattr(native, n) == values[n], (n, defines[n])


def test_gemm_desc_layout_matches_header():
    # the ctypes mirror must have the same size as the C struct (computed from the header fields)
    from pfd_b200 import native
    d = native.GemmDesc()
    # 1+3+3 int32 (=28, pad to 32) + 3 ptr + 9 int64 + 6 int32 + ptr + int32(+pad) + 2 int64 + float + int32
    # + 4 ptr + 6 int64 + 4 int32 (ndiv, cdiv, bn_force, tap_off) + stream ptr
    assert ctypes.sizeof(d) == 32 + 24 + 72 + 24 + 8 + 8 + 16 + 8 + 40 + 48 + 16 + 8
    # and the same field order as the header declares
    import re
    src = open(os.path.join(ROOT, "include", "pfd_b200.h")).read()
    start = "typedef struct pfd_gemm_desc {"
    body = src[src.index(start) + len(start):src.index("} pfd_gemm_desc;")]
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    names = []
    for decl in body.split(";"):
        decl = decl.strip()
        if not decl:
            continue
        for part in decl.split(","):
            m = re.search(r"(\w+)\s*(\[\w+\])?\s*$", part.strip())
            names.append(m.group(1))
    assert names == [f[0] for f in native.GemmDesc._fields_], (names, [f[0] for f in native.GemmDesc._fields_])


def test_bad_descriptor_is_rejected_without_gpu():
    from pfd_b200 import native
    lib = native.load()
    d = native.GemmDesc()
    d.nseg = 0
    assert lib.pfd_gemm_f16(ctypes.byref(d)) != 0
    assert b"nseg" in lib.pfd_last_error()
