"""CPU test: the Python binding and the library's layouts agree with include/fastga_b200.h and
fastga_b200/csrc/handles.h -- every C-ABI prototype, the two result structs, the raw record header and the
extension's counters."""
import ctypes as C
import os
import re

from fastga_b200 import lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _source(*path):
    """the file without its comments"""
    src = open(os.path.join(ROOT, *path)).read()
    return re.sub(r"//[^\n]*", "", re.sub(r"/\*.*?\*/", "", src, flags=re.S))


HEADER = _source("include", "fastga_b200.h")
HANDLES = _source("fastga_b200", "csrc", "handles.h")


def _c_kind(decl):
    """kind of a C parameter or return type: pointer, void or the scalar type"""
    if "*" in decl or "[" in decl:
        return "pointer"
    t = re.sub(r"\b(const|struct)\b", "", decl).split()
    return " ".join(t[:-1] if len(t) > 1 and t[-1] not in ("int", "long", "unsigned", "double", "float", "void")
                    else t)


_CTYPES_KIND = {C.c_int: "int", C.c_uint: "unsigned", C.c_longlong: "long long", C.c_double: "double",
                C.c_float: "float", None: "void"}


def _ctypes_kind(t):
    if t in (C.c_void_p, C.c_char_p) or (isinstance(t, type) and issubclass(t, C._Pointer)):
        return "pointer"
    return _CTYPES_KIND[t]


def header_prototypes():
    """{name: (return kind, [parameter kinds])} of every function the header declares"""
    protos = {}
    for ret, name, params in re.findall(r"([A-Za-z_][\w ]*?[\s*]+)(fgb_\w+)\s*\(([^)]*)\)\s*;", HEADER):
        params = [p.strip() for p in params.split(",")]
        if params == ["void"]:
            params = []
        assert name not in protos, name
        protos[name] = (_c_kind(ret.strip()), [_c_kind(p) for p in params])
    return protos


def _members(src, pattern):
    """(type, name) of the members of the struct whose body `pattern` captures, in order"""
    body = re.search(pattern, src, re.S).group(1)
    out = []
    for decl in body.split(";"):
        decl = decl.strip()
        if not decl:
            continue
        m = re.match(r"((?:unsigned\s+)?(?:long long|int|float|double|unsigned))\s+(.*)$", decl, re.S)
        out += [(m.group(1), n.strip()) for n in m.group(2).split(",")]
    return out


_SCALAR = {"long long": C.c_longlong, "int": C.c_int, "float": C.c_float, "unsigned long long": C.c_ulonglong}


def test_every_header_function_has_one_prototype_of_the_same_shape():
    protos = header_prototypes()
    assert len(protos) > 60
    assert set(lib.PROTOTYPES) == set(protos)
    for name, (ret, params) in protos.items():
        restype, argtypes = lib.PROTOTYPES[name]
        assert _ctypes_kind(restype) == ret, name
        assert [_ctypes_kind(a) for a in argtypes] == params, name


def test_result_structs_match_the_header():
    for cls, name in ((lib.RunStats, "fgb_run_stats"), (lib.Timings, "fgb_timings")):
        want = [(n, _SCALAR[t]) for t, n in _members(HEADER, r"typedef struct\s*\{([^{}]*)\}\s*%s\s*;" % name)]
        assert [(n, t) for n, t in cls._fields_] == want, name


def test_raw_record_dtype_matches_ovl_hdr():
    hdr = _members(HANDLES, r"struct ovl_hdr\s*\{(.*?)\}\s*;")
    assert [n for _, n in hdr] == list(lib.RAW_HDR_DT.names)
    assert all(t == "int" for t, _ in hdr)
    assert all(lib.RAW_HDR_DT[n].itemsize == 4 and lib.RAW_HDR_DT[n].kind == "i" for n in lib.RAW_HDR_DT.names)
    assert lib.RAW_HDR_DT.itemsize == 4 * len(hdr) == 40


def test_counter_names_match_ext_counters():
    fields = _members(HANDLES, r"struct ext_counters\s*\{(.*?)\}\s*;")
    assert len(lib.COUNTER_NAMES) == 16
    assert [n for _, n in fields] == list(lib.COUNTER_NAMES)
    assert all(t == "unsigned long long" for t, _ in fields)
