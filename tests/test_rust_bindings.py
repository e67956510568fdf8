"""CPU: the source-only Rust crate (integration/rust) stays in lock-step with include/cubecl_b200.h.

No Rust toolchain exists in this image, so the bindings are checked structurally instead of by compiling them:
  * src/sys.rs must be byte-identical to what tools/gen_rust_sys.py generates from the header NOW (every prototype, enum
    value, struct field and #define);
  * every `sys::b200_*` call in the hand-written safe layer (src/lib.rs) must name a header function and pass exactly as
    many arguments as the prototype has;
  * the safe layer's enums carry the header's numeric values.
"""
import importlib.util
import re
from pathlib import Path

from cubecl_b200._ffi import parse_header

ROOT = Path(__file__).resolve().parent.parent
spec = importlib.util.spec_from_file_location("gen_rust_sys", ROOT / "tools" / "gen_rust_sys.py")
gen = importlib.util.module_from_spec(spec)
spec.loader.exec_module(gen)

HEADER = (ROOT / "include" / "cubecl_b200.h").read_text()
SYS_RS = (ROOT / "integration" / "rust" / "src" / "sys.rs").read_text()
LIB_RS = (ROOT / "integration" / "rust" / "src" / "lib.rs").read_text()
LAUNCH_RS = (ROOT / "integration" / "rust" / "src" / "launch.rs").read_text()


def test_sys_rs_is_what_the_header_generates():
    assert SYS_RS == gen.render(HEADER), "run `python tools/gen_rust_sys.py` after changing include/cubecl_b200.h"


def test_every_header_function_is_bound_with_a_known_type():
    _, _, _, protos = parse_header(HEADER)
    names = [p[0] for p in protos]
    assert len(names) == len(set(names)) >= 51
    for name, _, args in protos:
        assert f"pub fn {name}(" in SYS_RS
        for _, ctype in args:
            assert ctype in gen.TYPES, f"{name}: no Rust mapping for C type '{ctype}'"


def _call_args(text, start):
    """number of top-level arguments of the call whose '(' is at text[start]"""
    depth, args, seen = 0, 0, False
    for ch in text[start:]:
        if ch in "([{":
            depth += 1
        elif ch in ")]}":
            depth -= 1
            if depth == 0:
                return args + (1 if seen else 0)
        elif ch == "," and depth == 1:
            args += 1
            seen = False
            continue
        elif depth >= 1 and not ch.isspace():
            seen = True
    raise AssertionError("unbalanced call")


def test_safe_layer_calls_match_the_prototypes():
    _, _, _, protos = parse_header(HEADER)
    arity = {name: len(args) for name, _, args in protos}
    calls = list(re.finditer(r"sys::(b200_\w+)\s*\(", LIB_RS))
    assert len(calls) >= 25
    for m in calls:
        name = m.group(1)
        assert name in arity, f"lib.rs calls sys::{name}, which the header does not declare"
        got = _call_args(LIB_RS, m.end() - 1)
        assert got == arity[name], f"sys::{name}: lib.rs passes {got} arguments, the header declares {arity[name]}"


def test_safe_layer_enums_carry_the_header_values():
    _, enums, _, _ = parse_header(HEADER)
    header = {ename: dict(items) for ename, items in enums}

    def rust_enum(name):
        body = re.search(r"pub enum " + name + r" \{(.*?)\}", LIB_RS, flags=re.S).group(1)
        return {k: int(v) for k, v in re.findall(r"(\w+) = (\d+)", body)}

    norm = lambda s: s.replace("_", "").lower()                                    # noqa: E731
    for rust, c, prefix in (("Status", "b200_status", "B200_ERR_"), ("DType", "b200_dtype", "B200_"),
                            ("ReduceOp", "b200_reduce_op", "B200_REDUCE_"), ("CommOp", "b200_comm_op", "B200_COMM_")):
        r = {norm(k): v for k, v in rust_enum(rust).items()}
        h = {norm(k[len(prefix):] if k.startswith(prefix) else k[len("B200_"):]): v for k, v in header[c].items()}
        assert r == h, (rust, r, h)


def test_launch_surface_only_uses_what_the_safe_layer_exports():
    # launch.rs (matmul::launch / reduce::launch over TensorHandle) is built on Context methods and crate-level items
    assert "pub mod launch;" in LIB_RS
    for m in re.finditer(r"ctx\.(\w+)\s*\(", LAUNCH_RS):
        decl = re.search(r"pub (?:unsafe )?fn " + m.group(1) + r"\s*\(([^{]*?)\)\s*->", LIB_RS, flags=re.S)
        assert decl, f"launch.rs calls Context::{m.group(1)}, which lib.rs does not define"
        want = len([a for a in decl.group(1).split(",") if a.strip() and "self" not in a])
        assert _call_args(LAUNCH_RS, m.end() - 1) == want, m.group(1)
    imported = re.search(r"use crate::\{(.*?)\};", LAUNCH_RS).group(1).split(",")
    for item in (i.strip() for i in imported):
        assert re.search(r"pub (?:struct|enum|fn|type) " + item + r"\b", LIB_RS) or re.search(r"pub use sys::\{[^}]*\b" + item + r"\b", LIB_RS), item
    # the shape rule is the one the Python mirror implements (shape.rs:489-517)
    assert "if l == r || r == 1" in LAUNCH_RS and "else if l == 1" in LAUNCH_RS
