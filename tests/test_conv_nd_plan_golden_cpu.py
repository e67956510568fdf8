"""CPU: the 3-D and transposed convolution entry points, and every failing call of the 2-D ones, replayed through a dry-run
planning context against golden/conv_nd_plan_golden.json.gz: the returned status, the full error message and the full plan
text must be byte-identical to the recorded ones.  Together with golden/conv_plan_golden.json.gz it pins the host-side
checks, their order, the messages, routing, operand staging, phase plans and launches of all convolution code;
golden/make_conv_nd_plan_golden.py writes it and holds the replay."""
import gzip
import json
import sys
from pathlib import Path

import pytest

sys.path.insert(0, str(Path(__file__).resolve().parent / "golden"))
from make_conv_nd_plan_golden import GOLDEN, replay  # noqa: E402

CASES = json.loads(gzip.decompress(GOLDEN.read_bytes()))["cases"]


@pytest.mark.parametrize("case", CASES, ids=[c["id"] for c in CASES])
def test_plan_matches_golden(case):
    got = replay(case["call"])
    assert (got["status"], got["error"]) == (case["status"], case["error"]), got
    assert got["plan"] == case["plan"]
