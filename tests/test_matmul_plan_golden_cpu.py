"""CPU: the matmul entry points (b200_matmul, _fused, _mixed, _scaled, _quantized, _quantized_fp8, _grouped and
_grouped_quantized_fp8) replayed through a dry-run
planning context against golden/matmul_plan_golden.json.gz: the returned status, the full error message and the full plan
text must be byte-identical to the recorded ones.  It pins the host-side checks, their order, the messages, routing, operand
staging, variant and stream-K choices, tensor maps and launches of the GEMM code; golden/make_matmul_plan_golden.py writes it
and holds the replay.  The recorded calls are grouped into one test per entry point, which names every call that differs."""
import gzip
import json
import sys
from pathlib import Path

import pytest

sys.path.insert(0, str(Path(__file__).resolve().parent / "golden"))
from make_matmul_plan_golden import GOLDEN, replay  # noqa: E402

CASES = json.loads(gzip.decompress(GOLDEN.read_bytes()))["cases"]
ENTRY_POINTS = sorted({c["call"]["fn"] for c in CASES})


@pytest.mark.parametrize("fn", ENTRY_POINTS)
def test_plans_match_golden(fn):
    cases = [c for c in CASES if c["call"]["fn"] == fn]
    assert cases
    differ = []
    for case in cases:
        got = replay(case["call"])
        want = {k: case[k] for k in ("status", "error", "plan")}
        if got != want:
            differ.append((case["id"], got, want))
    assert not differ, (f"{len(differ)} of {len(cases)} calls differ: {[d[0] for d in differ]}; "
                        f"first: {differ[0][0]}: got {differ[0][1]}, recorded {differ[0][2]}")
