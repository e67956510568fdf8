"""Extract the reference's plane-scan test vectors into scan_golden.json (read by tests/test_scan_*.py).

Needs a checkout of the reference (tracel-ai/cubecl @ 4057f39e):
    python tests/golden/make_scan_golden.py <path to the cubecl checkout>
test_plane_{inclusive,exclusive}_{sum,prod} (crates/cubecl-core/src/runtime_tests/plane.rs:191-405) compute their expectation
in the test from an input generator; this script checks that the sources still hold the generator, the starting value of the
expected loop, the vectorisations and the epsilon it records, and stores the expected arrays that loop produces, in its own
order, in f32.
"""
from __future__ import annotations

import json
import re
import sys
from pathlib import Path

import numpy as np

REF = Path(sys.argv[1]) if len(sys.argv) > 1 else None
OUT = Path(__file__).resolve().parent / "scan_golden.json"


def plane_scan_expected(op: str, exclusive: bool, vec: int) -> list[float]:
    """The expected loop of plane.rs test_plane_{in,ex}clusive_{sum,prod}, in its own order, in f32."""
    n = 32 * vec
    x = [np.float32(i) if op == "sum" else np.float32((0.5, 1.25, 1.75)[i % 3]) for i in range(n)]
    ident = np.float32(0.0 if op == "sum" else 1.0)
    exp = [ident] * n if exclusive else list(x)
    for k in range(1, 32):
        for k1 in range(k):
            for v in range(vec):
                exp[v + k * vec] = exp[v + k * vec] + x[v + k1 * vec] if op == "sum" else exp[v + k * vec] * x[v + k1 * vec]
    return [float(e) for e in exp]


def main() -> None:
    plane = (REF / "crates/cubecl-core/src/runtime_tests/plane.rs").read_text()
    eps = float(re.search(r"assert_equals_approx::<TestRuntime, F>\(&client, handle, expected, ([0-9.eE+-]+)\)", plane).group(1))
    gold = {"_generated_by": "tests/golden/make_scan_golden.py", "_reference": "tracel-ai/cubecl @ 4057f39e"}
    for kind, op in (("inclusive_sum", "sum"), ("exclusive_sum", "sum"), ("inclusive_prod", "prod"), ("exclusive_prod", "prod")):
        name = f"test_plane_{kind}"
        start = plane.index(f"pub fn {name}<")
        end = plane.index("\n}\n", start)
        body = plane[start:end]
        vecs = sorted({int(v) for v in re.findall(r"impl_" + name + r"\((\d+)\);", plane)})
        assert vecs == [1, 2, 4], (name, vecs)
        exclusive = kind.startswith("exclusive")
        init = ("vec![0.0; input.len()]" if op == "sum" else "vec![1.0; input.len()]") if exclusive else "input.clone();"
        assert "let mut expected = " + init in body, name
        if op == "sum":
            assert "x as f32" in body, name
        else:
            assert "0 => 0.5," in body and "1 => 1.25," in body and "2 => 1.75," in body, name
        gold[f"plane_{kind}"] = {
            "source": f"crates/cubecl-core/src/runtime_tests/plane.rs:{plane.count(chr(10), 0, start) + 1}-{plane.count(chr(10), 0, end) + 2}",
            "desc": (f"32 lanes x vec, {'value = flat index' if op == 'sum' else 'value = [0.5, 1.25, 1.75][flat index % 3]'}; "
                     f"lane k gets the {'exclusive' if exclusive else 'inclusive'} {op} over lanes of the same vector slot v "
                     f"(expected loops start from {'the identity' if exclusive else 'input[k]'}), assert_equals_approx"),
            "op": op, "exclusive": exclusive, "epsilon": eps, "vec_sizes": vecs,
            "generator": "index" if op == "sum" else "mod3:0.5,1.25,1.75",
            "expected": {str(v): plane_scan_expected(op, exclusive, v) for v in vecs},
        }
    OUT.write_text(json.dumps(gold, indent=1) + "\n")
    print("wrote", OUT, sorted(k for k in gold if not k.startswith("_")))


if __name__ == "__main__":
    if REF is None:
        raise SystemExit("usage: make_scan_golden.py <path to the cubecl checkout>")
    main()
