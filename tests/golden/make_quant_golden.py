"""Extract the reference's quantization vectors and constants into quant_golden.json (read by tests/test_quant_*.py).

Needs a checkout of the reference (tracel-ai/cubecl @ 4057f39e):
    python tests/golden/make_quant_golden.py <path to the cubecl checkout>
Only numbers are stored:
  * the inputs of the five symmetric known-answer tests of the quantized view (crates/cubecl-std/src/tests/view/quantized.rs):
    packed u32 words, value type, block size, block-scale dtype and values, per-tensor / global scale, and which of the
    test's expectation formulas applies;
  * the scale probe grid of the host/device round-up differential test (crates/cubecl-std/src/tests/round.rs) and the
    dtypes it runs;
  * ScaleDtype::max_representable / f32_grid and QuantValue::range() (crates/cubecl-common/src/quant/scheme.rs).
"""
from __future__ import annotations

import json
import re
import sys
from pathlib import Path

import numpy as np

REF = Path(sys.argv[1]) if len(sys.argv) > 1 else None
OUT = Path(__file__).resolve().parent / "quant_golden.json"

KATS = {   # test fn -> expectation formula of its body
    "test_quantized_per_tensor_int": "int_range_times_scale",
    "test_quantized_per_tensor_fp4": "e2m1_code_times_scale",
    "test_quantized_global_scale": "global_times_block_times_int",
    "test_quantized_two_level_int": "global_times_block_times_int",
    "test_quantized_two_level_ue4m3": "global_times_block_times_int",
}


def fn_body(text: str, name: str) -> tuple[str, int, int]:
    start = text.index(f"pub fn {name}<")
    end = text.index("\n}\n", start)
    return text[start:end], text.count("\n", 0, start) + 1, text.count("\n", 0, end) + 2


def main() -> None:
    view = (REF / "crates/cubecl-std/src/tests/view/quantized.rs").read_text()
    scheme = (REF / "crates/cubecl-common/src/quant/scheme.rs").read_text()
    rnd = (REF / "crates/cubecl-std/src/tests/round.rs").read_text()
    gold = {"_generated_by": "tests/golden/make_quant_golden.py", "_reference": "tracel-ai/cubecl @ 4057f39e", "kats": {}}

    for name, formula in KATS.items():
        body, l0, l1 = fn_body(view, name)
        words = [int(w, 16) for w in re.search(r"u32::as_bytes\(&\[(0x[0-9A-F]+), (0x[0-9A-F]+)\]\)", body).groups()]
        value = re.search(r"\.with_value\(QuantValue::(\w+)\)", body).group(1)
        kat = {"source": f"crates/cubecl-std/src/tests/view/quantized.rs:{l0}-{l1}", "words": words, "value": value,
               "formula": formula, "len": 16}
        blk = re.search(r"let block = (\d+);", body)
        if blk:
            kat["block"] = int(blk.group(1))
            kat["block_scale"] = re.search(r"\.per_block\(\[block as u8\], ScaleDtype::(\w+)\)", body).group(1)
            assert ".per_tensor(ScaleDtype::F32)" in body, name
            kat["global_scale_pow2"] = int(re.search(r"let global_scale = 2f32\.powi\((-?\d+)\);", body).group(1))
            pw = re.search(r"let block_scales = \[2f32\.powi\((-?\d+)\), 2f32\.powi\((-?\d+)\)\];", body)
            if pw:
                kat["block_scales"] = [float(np.ldexp(1.0, int(e))) for e in pw.groups()]
            else:
                e4 = re.search(r"let block_scales = \[e4m3::from_f32\(([0-9.]+)\), e4m3::from_f32\(([0-9.]+)\)\];", body)
                kat["block_scales"] = [float(v) for v in e4.groups()]
            assert "(i as f32 - 8.0)" in body and "block_scales[i / block]" in body, name
        else:
            kat["block"] = 0
            kat["tensor_scale"] = float(re.search(r"let scales = client\.create_from_slice\(f32::as_bytes\(&\[([0-9.]+)\]\)\);", body).group(1))
            assert ("(-8..=7)" in body) == (formula == "int_range_times_scale"), name
            assert ("e2m1::from_bits" in body) == (formula == "e2m1_code_times_scale"), name
        gold["kats"][name] = kat

    # the probe grid of test_round_up_matches_host
    m = re.search(r"\((-?\d+)\.\.(-?\d+)\)\s*\.flat_map\(\|exp\| \((\d+)\.\.(\d+)\)\.map\(move \|step\| \(step as f32 / ([0-9.]+)\)", rnd)
    mults = re.search(r"scales\.extend\(\[max \* ([0-9.]+), max \* ([0-9.]+), max, max \* ([0-9.]+), f32::MAX\]\);", rnd)
    dtypes = re.findall(r"round_up_matches_host_\w+ => (\w+)", rnd)
    gold["round_up_grid"] = {
        "source": "crates/cubecl-std/src/tests/round.rs:22-28",
        "exp": [int(m.group(1)), int(m.group(2))], "step": [int(m.group(3)), int(m.group(4))], "step_div": float(m.group(5)),
        "max_multipliers": [float(mults.group(1)), float(mults.group(2)), 1.0, float(mults.group(3))], "f32_max": True,
        "dtypes": dtypes,
    }

    # ScaleDtype constants: max_representable and the f32 grid (bit step, subnormal range)
    assert "ScaleDtype::UE8M0 => f32::from_bits(0x7F00_0000)" in scheme and "ScaleDtype::UE4M3 => 448.0" in scheme
    assert "half::f16::MAX.to_f32()" in scheme and "half::bf16::MAX.to_f32()" in scheme and "ScaleDtype::F32 => f32::MAX" in scheme
    assert "bit_step: bit_step(4)" in scheme and "min_normal: 0.015625" in scheme and "spacing: 0.001953125" in scheme
    assert "bit_step(half::f16::MANTISSA_DIGITS)" in scheme and "bit_step(half::bf16::MANTISSA_DIGITS)" in scheme
    f16_min_normal, f16_spacing = float(np.finfo(np.float16).tiny), float(np.float16(np.finfo(np.float16).smallest_subnormal))
    gold["scale_dtypes"] = {
        "F32": {"max": float(np.finfo(np.float32).max)},
        "F16": {"max": float(np.finfo(np.float16).max), "bit_step": 1 << (24 - 11), "min_normal": f16_min_normal, "spacing": f16_spacing},
        "BF16": {"max": float(np.uint32(0x7F7F0000).view(np.float32)), "bit_step": 1 << (24 - 8)},
        "UE4M3": {"max": 448.0, "bit_step": 1 << (24 - 4), "min_normal": 0.015625, "spacing": 0.001953125},
        "UE8M0": {"max": float(np.uint32(0x7F000000).view(np.float32))},
    }

    # QuantValue::range()
    body = scheme[scheme.index("pub fn range(&self)"):]
    body = body[:body.index("\n    }\n")]
    rng = {}
    for v, lo, hi in re.findall(r"QuantValue::(\w+) => \(([^,]+), ([^)]+)\)", body):
        def num(s):
            s = s.strip()
            return {"i8::MIN as f32": -128.0, "i8::MAX as f32": 127.0, "-i8::MAX as f32": -127.0}.get(s, None) if "i8" in s else float(s)
        rng[v] = [num(lo), num(hi)]
    assert len(rng) == 9, rng
    gold["range"] = rng
    OUT.write_text(json.dumps(gold, indent=1) + "\n")
    print("wrote", OUT, sorted(gold["kats"]))


if __name__ == "__main__":
    if REF is None:
        raise SystemExit("usage: make_quant_golden.py <path to the cubecl checkout>")
    main()
