"""In-tree build of the native pieces (no JIT cache, no pip install):

  csrc/*.cu  --nvcc -cubin, sm_90a-->  build/*.cubin  --.incbin-->  lib/libcubecl_b200.so  (host: g++, dlopen's libcuda)

The cubins are PREBUILT images loaded with cuModuleLoadData at b200_init(); nothing is compiled at run time
(the reference's NVRTC step, crates/cubecl-cuda/src/compute/context.rs:141-317, is what this replaces).

`python -m cubecl_b200.build` or `__graft_entry__.build()` runs it; nvcc cross-compiles without a GPU.
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys
from pathlib import Path

PKG = Path(__file__).resolve().parent
ROOT = PKG.parent
CSRC = PKG / "csrc"
BUILD = PKG / "build"
LIBDIR = PKG / "lib"
LIB = LIBDIR / "libcubecl_b200.so"

# tag -> (source, extra nvcc flags); the GEMM source is split in eleven cubins so the parts compile in parallel
CUBINS = {"gemm": ("gemm_wgmma.cu", ["-DGEMM_PART=0"]), "gemm_b": ("gemm_wgmma.cu", ["-DGEMM_PART=1"]),
          "gemm_c": ("gemm_wgmma.cu", ["-DGEMM_PART=2"]), "reduce": ("reduce.cu", []), "aux": ("aux_kernels.cu", []),
          "quant": ("quant.cu", []), "gemm_q": ("gemm_wgmma.cu", ["-DGEMM_PART=3"]),
          "quant_mm": ("quant.cu", ["-DQUANT_PART=1"]), "gemm_conv": ("gemm_wgmma.cu", ["-DGEMM_PART=4"]),
          "gemm_convbwd": ("gemm_wgmma.cu", ["-DGEMM_PART=5"]), "conv_grouped": ("conv_grouped.cu", []),
          "gemm_conv3d": ("gemm_wgmma.cu", ["-DGEMM_PART=6"]), "gemm_convt": ("gemm_wgmma.cu", ["-DGEMM_PART=7"]),
          "gemm_grouped": ("gemm_wgmma.cu", ["-DGEMM_PART=8"]), "gemm_qf8": ("gemm_wgmma.cu", ["-DGEMM_PART=9"]),
          "gemm_grouped_qf8": ("gemm_wgmma.cu", ["-DGEMM_PART=10"]),
          "attention": ("attention.cu", []), "attention_bwd": ("attention_bwd.cu", []),
          "attention_kv": ("attention_kv.cu", []), "attention_varlen": ("attention.cu", ["-DATTN_VARLEN"]),
          "attention_varlen_bwd": ("attention_bwd.cu", ["-DATTN_VARLEN"]),
          "attention_kv_fp8": ("attention_kv.cu", ["-DATTN_KV_FP8"]),
          "attention_paged": ("attention.cu", ["-DATTN_VARLEN", "-DATTN_PAGED"]),
          "attention_paged_fp8": ("attention.cu", ["-DATTN_VARLEN", "-DATTN_PAGED", "-DATTN_PAGED_FP8"])}
NVCC_FLAGS = ["-cubin", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17"]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and Path(cand).exists():
            return cand
    raise RuntimeError("nvcc not found: the CUDA kernels cannot be built")


def _cuda_include() -> str:
    for cand in (os.environ.get("CUDA_HOME"), "/usr/local/cuda"):
        if cand and (Path(cand) / "include" / "cuda.h").exists():
            return str(Path(cand) / "include")
    raise RuntimeError("cuda.h not found")


def _digest(paths) -> str:
    h = hashlib.sha256()
    for p in sorted(paths):
        h.update(p.name.encode())
        h.update(p.read_bytes())
    return h.hexdigest()


def _run(cmd, **kw):
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, **kw)
    if r.returncode != 0:
        raise RuntimeError("build step failed: " + " ".join(map(str, cmd)) + "\n" + r.stdout)
    return r.stdout


def build(force: bool = False, verbose: bool = False) -> Path:
    """Build lib/libcubecl_b200.so if sources changed. Returns the library path."""
    BUILD.mkdir(exist_ok=True)
    LIBDIR.mkdir(exist_ok=True)
    sources = [p for p in CSRC.iterdir() if p.suffix in (".cu", ".cuh", ".cpp", ".h")]
    sources += [ROOT / "include" / "cubecl_b200.h", ROOT / "include" / "cubecl_b200.hpp", ROOT / "examples" / "sum_things.cpp"]
    stamp = BUILD / "stamp.txt"
    digest = _digest(sources)
    if not force and LIB.exists() and stamp.exists() and stamp.read_text() == digest:
        return LIB
    nvcc = _nvcc()

    # every cubin is rebuilt only when ITS inputs changed (source, the shared headers, the flags): editing reduce.cu does not
    # cost the five minutes of ptxas the GEMM instantiations take
    def inputs_digest(src, extra):
        h = hashlib.sha256(" ".join(NVCC_FLAGS + list(extra)).encode())
        for f in (CSRC / src, CSRC / "ptx.cuh", CSRC / "epilogue.cuh", CSRC / "attention.cuh", CSRC / "kernel_params.h",
                  ROOT / "include" / "cubecl_b200.h"):
            h.update(f.read_bytes())
        return h.hexdigest()

    def compile_one(item):
        tag, (src, extra) = item
        out, mark = BUILD / f"{tag}.cubin", BUILD / f"{tag}.stamp"
        want = inputs_digest(src, extra)
        if not force and out.exists() and mark.exists() and mark.read_text() == want:
            return f"{tag}: up to date"
        log = _run([nvcc, *NVCC_FLAGS, *extra, "-Xptxas", "-v", str(CSRC / src), "-o", str(out)])
        (BUILD / f"{tag}.ptxas.log").write_text(log)
        mark.write_text(want)
        return log

    from concurrent.futures import ThreadPoolExecutor
    with ThreadPoolExecutor(max_workers=len(CUBINS)) as pool:
        for log in pool.map(compile_one, CUBINS.items()):
            if verbose:
                print(log)
    # embed the cubins with .incbin (64-byte aligned, begin/end symbols)
    asm = [".section .rodata\n"]
    for tag in CUBINS:
        asm.append(
            f".global b200_cubin_{tag}\n.global b200_cubin_{tag}_end\n.balign 64\n"
            f"b200_cubin_{tag}:\n.incbin \"{BUILD / (tag + '.cubin')}\"\nb200_cubin_{tag}_end:\n.byte 0\n"
        )
    asm.append('.section .note.GNU-stack,"",@progbits\n')
    embed = BUILD / "embed.S"
    embed.write_text("".join(asm))
    _run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-I", _cuda_include(),
          str(CSRC / "capi.cpp"), str(embed), "-ldl", "-lpthread", "-o", str(LIB)])
    # C++ host-layer example (include/cubecl_b200.hpp): compiled here so the header cannot rot; run on the GPU box by
    # tests/test_cpp_host_gpu.py
    _run(["g++", "-O2", "-std=c++17", "-Wall", "-I", str(ROOT / "include"), str(ROOT / "examples" / "sum_things.cpp"),
          "-L", str(LIBDIR), "-lcubecl_b200", f"-Wl,-rpath,{LIBDIR}", "-Wl,-rpath,$ORIGIN", "-o", str(LIBDIR / "sum_things_cpp")])
    stamp.write_text(digest)
    return LIB


if __name__ == "__main__":
    path = build(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print(path)
