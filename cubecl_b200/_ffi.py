"""ctypes binding of include/cubecl_b200.h, derived from the header when this module is imported.

Every `#define B200_*` and enum item becomes a module constant without its `B200_` prefix (F32, REDUCE_SUM, QV_Q8F, ...),
every struct a ctypes.Structure named in CamelCase without `b200_` (b200_quant_operand -> QuantOperand), and every prototype
a row of SIGNATURES.  So the header is the only copy of the ABI; a C type the maps below do not know fails the import.

Loading this module never needs a GPU (the library dlopen's libcuda lazily), so the CPU test-suite can check that the
library loads and exports every declared symbol.  Any compute call without a GPU fails loudly with B200Error -- there is
no CPU fallback on the product path.
"""
from __future__ import annotations

import ctypes as C
import re
from pathlib import Path

PKG = Path(__file__).resolve().parent
LIB_PATH = PKG / "lib" / "libcubecl_b200.so"
HEADER_PATH = PKG.parent / "include" / "cubecl_b200.h"

STATUS_NAMES = {
    0: "Ok", 1: "CompilationError", 2: "OutOfMemory", 3: "TooManyResources", 4: "Unknown", 5: "IoError",
    6: "InvalidArgument", 7: "Unsupported", 8: "NoDevice", 9: "Communication", 10: "ServerUnhealthy",
}


class B200Error(RuntimeError):
    """Mirrors LaunchError / ServerError (crates/cubecl-runtime/src/server/base.rs:177-272)."""

    def __init__(self, status: int, message: str):
        super().__init__(f"{STATUS_NAMES.get(status, status)}: {message}")
        self.status = status
        self.kind = STATUS_NAMES.get(status, str(status))


def strip_comments(text: str) -> str:
    return re.sub(r"/\*.*?\*/", " ", text, flags=re.S)


def parse_header(text: str):
    """(consts, enums, structs, protos) of the header text:
      consts  [(name, value)] of the `#define B200_* <n>` lines;
      enums   [(enum, [(item, value)])];
      structs [(struct, [(field, C type)])], a `char x[N]` field typed "char[N]";
      protos  [(function, return type, [(parameter, C type)])], a pointer spelt "T*" (no space before the '*')."""
    body = strip_comments(text)
    enums, structs, protos, consts = [], [], [], []
    for m in re.finditer(r"#define\s+(B200_[A-Z0-9_]+)\s+(\d+)", body):
        consts.append((m.group(1), int(m.group(2))))
    for m in re.finditer(r"typedef\s+enum\s+(\w+)\s*\{(.*?)\}\s*\w+\s*;", body, flags=re.S):
        items = [(k, int(v)) for k, v in re.findall(r"(B200_[A-Z0-9_]+)\s*=\s*(\d+)", m.group(2))]
        enums.append((m.group(1), items))
    for m in re.finditer(r"typedef\s+struct\s+(\w+)\s*\{(.*?)\}\s*\w+\s*;", body, flags=re.S):
        fields = []
        for decl in m.group(2).split(";"):
            decl = " ".join(decl.split())
            if not decl:
                continue
            arr = re.match(r"char (\w+)\[(\d+)\]$", decl)
            if arr:
                fields.append((arr.group(1), f"char[{arr.group(2)}]"))
                continue
            ctype, names = decl.split(" ", 1)
            for name in names.split(","):
                fields.append((name.strip(), ctype))
        structs.append((m.group(1), fields))
    for m in re.finditer(r"(?m)^(int|const char\*)\s+(b200_\w+)\s*\(([^;{]*?)\)\s*;", body, flags=re.S):
        ret, name, params = m.group(1), m.group(2), " ".join(m.group(3).split())
        args = []
        if params != "void":
            for p in params.split(","):
                p = p.strip()
                pm = re.match(r"(.*?)(\w+)$", p)
                ctype = pm.group(1).strip().replace(" *", "*")
                args.append((pm.group(2), ctype))
        protos.append((name, ret, args))
    return consts, enums, structs, protos


# C type -> ctypes type, for struct fields and parameters alike.  Handles are opaque pointers; below, every enum is added as
# c_int (the C ABI passes enums as int) and every struct as its Structure.
_CTYPES = {
    "int": C.c_int, "int32_t": C.c_int32, "uint32_t": C.c_uint32, "int64_t": C.c_int64, "uint64_t": C.c_uint64,
    "b200_dptr": C.c_uint64, "size_t": C.c_size_t, "float": C.c_float, "double": C.c_double, "char*": C.c_char_p,
    "void*": C.c_void_p, "b200_ctx*": C.c_void_p, "b200_stream": C.c_void_p, "b200_event": C.c_void_p,
}


def _ctype(spelling: str):
    """The ctypes type of a C type as parse_header spells it: T* is POINTER(T) unless the map names T* itself."""
    t = spelling.removeprefix("const ")
    if t in _CTYPES:
        return _CTYPES[t]
    if t.endswith("*"):
        return C.POINTER(_ctype(t[:-1]))
    arr = re.fullmatch(r"char\[(\d+)\]", t)
    if arr:
        return C.c_char * int(arr.group(1))
    raise TypeError(f"{HEADER_PATH.name}: no ctypes mapping for the C type '{spelling}'")


def _structure(name: str, fields):
    cls = type("".join(w.capitalize() for w in name.removeprefix("b200_").split("_")), (C.Structure,),
               {"_fields_": [(f, _ctype(t)) for f, t in fields]})
    _CTYPES[name] = cls
    return cls


_consts, _enums, _structs, _protos = parse_header(HEADER_PATH.read_text())
globals().update((name.removeprefix("B200_"), value) for name, value in _consts + [i for _, items in _enums for i in items])
_CTYPES.update((name, C.c_int) for name, _ in _enums)
STRUCTS = {name: _structure(name, fields) for name, fields in _structs}   # header order: a struct precedes those embedding it
globals().update((cls.__name__, cls) for cls in STRUCTS.values())
SIGNATURES = {name: (_ctype(ret), [_ctype(t) for _, t in args]) for name, ret, args in _protos}   # name -> (restype, argtypes)

_lib = None


def load() -> C.CDLL:
    """dlopen the in-tree library; raise if it is missing (the product path never degrades to a CPU implementation)."""
    global _lib
    if _lib is not None:
        return _lib
    if not LIB_PATH.exists():
        # a fresh checkout (built artefacts are git-ignored): build in-tree once; nvcc cross-compiles without a GPU
        try:
            from . import build as _build
            _build.build()
        except Exception as e:  # noqa: BLE001
            raise B200Error(1, f"{LIB_PATH} is missing and could not be built ({e}). There is no CPU fallback.") from e
    lib = C.CDLL(str(LIB_PATH))
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the .so does not export what the header declares
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(status: int) -> None:
    if status != 0:
        msg = load().b200_last_error()
        raise B200Error(status, msg.decode() if msg else "")


def u64_array(values) -> C.Array:
    values = [int(v) for v in values]
    return (C.c_uint64 * len(values))(*values)


def int_array(values) -> C.Array:
    values = [int(v) for v in values]
    return (C.c_int * len(values))(*values)
