"""CPU: every attention entry point (dense forward and backward, KV cache and its write, varlen forward and backward) replayed
through a dry-run planning context against golden/attention_plan_golden.json.gz: the returned status, the entry-point prefix of
the error message and the full plan text must be byte-identical to the recorded ones.  The fixture pins the host-side checks,
operand staging and launches of the attention code; golden/make_attention_plan_golden.py writes it and holds the replay."""
import gzip
import json
import sys
from pathlib import Path

import pytest

sys.path.insert(0, str(Path(__file__).resolve().parent / "golden"))
from make_attention_plan_golden import GOLDEN, replay  # noqa: E402

CASES = json.loads(gzip.decompress(GOLDEN.read_bytes()))["cases"]


@pytest.mark.parametrize("case", CASES, ids=[c["id"] for c in CASES])
def test_plan_matches_golden(case):
    got = replay(case["call"])
    assert (got["status"], got["error"]) == (case["status"], case["error"]), got
    assert got["plan"] == case["plan"]
