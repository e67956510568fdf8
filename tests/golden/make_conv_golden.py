"""Extract the reference's im2col known-answer test into conv_golden.json (read by tests/test_conv_*.py).

Needs a checkout of the reference (tracel-ai/cubecl @ 4057f39e):
    python tests/golden/make_conv_golden.py <path to the cubecl checkout>
test_tensormap_load_im2col (crates/cubecl-core/src/runtime_tests/tensormap.rs:212-300) loads x = 1..N*H*W*C as [N, H, W, C]
through a 4-D im2col tensor map and compares the [KH*KW, pixels, C] result with a table of pixel numbers (0 = padding, p = the
p-th input pixel, 1-based).  This script reads the shape, kernel, padding and that table from the source and stores them.
"""
from __future__ import annotations

import json
import re
import sys
from pathlib import Path

REF = Path(sys.argv[1]) if len(sys.argv) > 1 else None
OUT = Path(__file__).resolve().parent / "conv_golden.json"


def main() -> None:
    src = (REF / "crates/cubecl-core/src/runtime_tests/tensormap.rs").read_text()
    body = src[src.index("pub fn test_tensormap_load_im2col"):]
    body = body[:body.index("\npub fn ")]
    val = {k: int(re.search(rf"let {k} = (-?\d+);", body).group(1)) for k in ("n", "h", "w", "c", "kernel_h", "kernel_w",
                                                                               "pad_h", "pad_w", "out_h", "out_w")}
    rows = [json.loads("[" + r + "]") for r in re.findall(r"(?:vec!|extend\()\[([0-9, ]+)\]", body)]
    assert len(rows) == val["kernel_h"] * val["kernel_w"] and all(len(r) == val["n"] * val["out_h"] * val["out_w"] for r in rows)
    gold = {"_generated_by": "tests/golden/make_conv_golden.py", "_reference": "tracel-ai/cubecl @ 4057f39e",
            "_source": "crates/cubecl-core/src/runtime_tests/tensormap.rs: test_tensormap_load_im2col",
            "im2col_kat": {**val, "x": "1..n*h*w*c as [n, h, w, c]",
                           "expected_pixels": rows}}
    OUT.write_text(json.dumps(gold, indent=1) + "\n")
    print(f"wrote {OUT}")


if __name__ == "__main__":
    main()
