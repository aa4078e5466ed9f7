"""The ctypes mirror of the C ABI (linetr_b200/_native.py) against include/linetr_b200.h and
include/linetr_b200_debug.h: every struct's fields, widths, pointee types, offsets and size, every ltr_* prototype's
argument and return types, and every constant the binding repeats.  A mismatch would otherwise only show as garbage
read on the GPU.  CPU only; offsets, sizes and macro values come from the host C compiler and are skipped without one."""
import ctypes as C
import os
import re
import shutil
import subprocess

import pytest

from linetr_b200 import _native as N

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INCLUDE = os.path.join(ROOT, "include")
HEADERS = ("linetr_b200.h", "linetr_b200_debug.h")
# what the ABI fixes of a C scalar type: integer or floating point, and its width
SCALARS = {"int": "int32", "int32_t": "int32", "int64_t": "int64", "uint64_t": "int64", "uint8_t": "int8",
           "float": "float32", "double": "float64"}
WORKSPACE_SIZES = ((0, 0, 0), (1, 480, 640), (256, 480, 640), (3, 7, 5), (1000, 1200, 1600))   # the last > 2^31


def _text(header):
    """A header without comments."""
    return re.sub(r"/\*.*?\*/|//[^\n]*", " ", open(os.path.join(INCLUDE, header)).read(), flags=re.S)


def _declarations(header):
    """The header's declarations, split at ';', '{' and '}', without preprocessor lines."""
    return re.split(r"[;{}]", re.sub(r"^\s*#.*$", "", _text(header), flags=re.M))


def _kind(c_type, declarator=""):
    """'pointer', None (void) or SCALARS[type] of a declaration split into its type and declarator."""
    if "*" in c_type + declarator or "[" in declarator:
        return "pointer"
    t = " ".join(w for w in c_type.split() if w not in ("const", "struct"))
    return None if t == "void" else SCALARS[t]


def _pointee(c_type, declarator):
    """SCALARS[T] of a `[const] T*` declaration with a scalar T, else None (void*, char*, struct pointers, pointers to
    pointers and arrays)."""
    t = " ".join(w for w in c_type.split() if w not in ("const", "struct"))
    return SCALARS.get(t) if declarator.count("*") == 1 and "[" not in declarator else None


def _ctype_kind(t):
    if t is None:
        return None
    if t in (C.c_void_p, C.c_char_p) or issubclass(t, C._Pointer):
        return "pointer"
    return ("float" if t._type_ in "fdg" else "int") + str(8 * C.sizeof(t))


def _ctype_pointee(st, f, t):
    """The kind of what field f of mirror st (type t) points to: its tag in st._pointees_ (_native.F32P ...) or c_T of
    POINTER(c_T), else None."""
    if f in getattr(st, "_pointees_", {}):
        return _ctype_kind(st._pointees_[f])
    if issubclass(t, C._Pointer) and issubclass(t._type_, C._SimpleCData):
        return _ctype_kind(t._type_)
    return None


def _declarators(decl):
    """'const int32_t* a, b[4]' -> [('a', kind, pointee), ('b', kind, pointee)]."""
    m = re.fullmatch(r"\s*((?:const\s+|struct\s+|unsigned\s+|long\s+)*\w+)(.*?)\s*", decl, re.S)
    out = []
    for d in m.group(2).split(","):
        p = re.fullmatch(r"([\s*]*(?:const\s*\*?\s*)*)(\w+)\s*(\[\w*\])?\s*", d)
        declarator = p.group(1) + (p.group(3) or "")
        out.append((p.group(2), _kind(m.group(1), declarator), _pointee(m.group(1), declarator)))
    return out


def _structs():
    """{name: [(field, kind, pointee)]} of every `typedef struct {...} Name;` of the headers, fields in order."""
    out = {}
    for h in HEADERS:
        for body, name in re.findall(r"typedef\s+struct\s*\{([^{}]*)\}\s*(\w+)\s*;", _text(h)):
            out[name] = [f for decl in body.split(";") if decl.strip() for f in _declarators(decl)]
    return out


def _prototypes():
    """{name: (return kind, [argument kinds])} of every ltr_* function the headers declare."""
    out = {}
    for h in HEADERS:
        for decl in _declarations(h):
            m = re.fullmatch(r"\s*(.*?)\b(ltr_\w+)\s*\((.*)\)\s*", decl, re.S)
            if m:
                args = [] if m.group(3).strip() == "void" else m.group(3).split(",")
                out[m.group(2)] = (_kind(m.group(1)), [k for a in args for _, k, _ in _declarators(a)])
    return out


STRUCTS = _structs()
PROTOS = _prototypes()


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    """{key: value} printed by a C program built against the header: 'Struct.field' offsets, 'Struct' sizes and
    'ws n h w' LTR_PHOTOMETRIC_WORKSPACE_BYTES values; None without a host C compiler."""
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        return None
    lines = []
    for name, fields in STRUCTS.items():
        lines += [f'  printf("{name}.{f} %zu\\n", offsetof({name}, {f}));' for f, _, _ in fields]
        lines.append(f'  printf("{name} %zu\\n", sizeof({name}));')
    for n, h, w in WORKSPACE_SIZES:
        lines.append(f'  printf("ws {n} {h} {w} %lld\\n", (long long)LTR_PHOTOMETRIC_WORKSPACE_BYTES({n}, {h}, {w}));')
    td = tmp_path_factory.mktemp("abi")
    src, exe = str(td / "abi.c"), str(td / "abi")
    with open(src, "w") as f:
        f.write('#include <stdio.h>\n#include <stddef.h>\n#include "linetr_b200.h"\nint main(void) {\n'
                + "\n".join(lines) + "\n  return 0;\n}\n")
    subprocess.check_call([cc, "-I", INCLUDE, "-o", exe, src])
    out = subprocess.check_output([exe]).decode().splitlines()
    return {k: int(v) for k, v in (ln.rsplit(" ", 1) for ln in out)}


def test_every_struct_and_prototype_is_mirrored():
    mirrored = {k for k, v in vars(N).items() if isinstance(v, type) and issubclass(v, C.Structure)}
    assert mirrored == set(STRUCTS), mirrored ^ set(STRUCTS)
    table = {**N.PROTOTYPES, **N.DEBUG_PROTOTYPES}
    assert set(table) == set(PROTOS), set(table) ^ set(PROTOS)


@pytest.mark.parametrize("name", list(STRUCTS))
def test_struct_layout_matches_header(name, compiled):
    st = getattr(N, name)
    want = STRUCTS[name]
    got = [(f, _ctype_kind(t), _ctype_pointee(st, f, t)) for f, t in st._fields_]
    assert [f for f, _, _ in got] == [f for f, _, _ in want], f"{name}: fields differ from the header"
    for (f, k, e), (_, g, ge) in zip(want, got):
        assert g == k, f"{name}.{f}: {g} in the binding, {k} in the header"
        assert ge == e, f"{name}.{f}: points to {ge} in the binding, {e} in the header"
    if compiled is None:
        pytest.skip("no host C compiler for the offsetof check")
    for f, _, _ in want:
        assert getattr(st, f).offset == compiled[f"{name}.{f}"], f"{name}.{f}: offset differs from the header"
    assert C.sizeof(st) == compiled[name], f"{name}: size differs from the header"


@pytest.mark.parametrize("name", sorted(PROTOS))
def test_prototype_matches_header(name):
    restype, argtypes = {**N.PROTOTYPES, **N.DEBUG_PROTOTYPES}[name]
    ret, args = PROTOS[name]
    assert _ctype_kind(restype) == ret, f"{name}: returns {_ctype_kind(restype)} in the binding, {ret} in the header"
    assert len(argtypes) == len(args), f"{name}: {len(argtypes)} arguments in the binding, {len(args)} in the header"
    for i, (t, k) in enumerate(zip(argtypes, args)):
        assert _ctype_kind(t) == k, f"{name}: argument {i} is {_ctype_kind(t)} in the binding, {k} in the header"


def test_routed_entries_take_device_and_stream():
    """_ops._call appends (device, stream) to its arguments, and ctypes passes surplus arguments without complaint, so
    every entry routed through it must end its prototype with them."""
    pkg = os.path.join(ROOT, "linetr_b200")
    src = "".join(open(os.path.join(pkg, f)).read() for f in sorted(os.listdir(pkg)) if f.endswith(".py"))
    routed = set(re.findall(r"\b(?:_call|_match|call_struct)\(\s*\"(ltr_\w+)\"", src))
    assert {"ltr_match", "ltr_tokenize_batch", "ltr_gather_wait"} <= routed
    decls = "".join(_declarations("linetr_b200.h"))
    for name in routed:
        args = re.search(r"\b" + name + r"\s*\(([^()]*)\)", decls).group(1)
        assert re.search(r"int32_t\s+device\s*,\s*void\s*\*\s*stream\s*$", args), \
            f"{name} does not end with (int32_t device, void* stream) but is called through _ops._call"


def test_constants_match_header(compiled):
    defined = dict(re.findall(r"^\s*#define\s+(LTR_\w+)\s+(\d+)\s*$", _text("linetr_b200.h"), flags=re.M))
    for macro, value in (("LTR_ABI_VERSION", N.ABI_VERSION), ("LTR_GATHER_SLOTS", N.GATHER_SLOTS),
                         ("LTR_LAYOUT_ROWS", N.LAYOUT_ROWS), ("LTR_LAYOUT_CHANNEL_FIRST", N.LAYOUT_CHANNEL_FIRST),
                         ("LTR_PHOTOMETRIC_PARAMS", N.PHOTOMETRIC_PARAMS),
                         ("LTR_PHOTOMETRIC_MAX_KSIZE", N.PHOTOMETRIC_MAX_KSIZE)):
        assert int(defined[macro]) == value, f"{macro}: {value} in the binding, {defined[macro]} in the header"
    if compiled is None:
        pytest.skip("no host C compiler for LTR_PHOTOMETRIC_WORKSPACE_BYTES")
    for n, h, w in WORKSPACE_SIZES:
        assert N.photometric_workspace_bytes(n, h, w) == compiled[f"ws {n} {h} {w}"], \
            f"photometric_workspace_bytes{(n, h, w)} differs from LTR_PHOTOMETRIC_WORKSPACE_BYTES"
