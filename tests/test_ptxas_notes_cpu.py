"""The wgmma chains of the convolution kernels stay asynchronous: ptxas reports, in the -Xptxas -v output that
holocron_b200/csrc/build.py keeps in csrc/build/<unit>.log, when it has to serialise wgmma instructions
(C7511: not enough registers for the pipeline; C7520: a warpgroup arrive it inserted on a divergent path) or to insert
warpgroup arrives around accumulator accesses (C7519). Any of these puts every MMA of the kernel behind the previous
one. Spills are checked as well: they would put the accumulators in local memory. The pooling, attention, involution and
lambda units hold no wgmma; their register-heavy kernels (SAM backward, the lambda output and dq kernels at their
launch-bound cap) are checked for spills."""
import re
from pathlib import Path

import pytest

BUILD = Path(__file__).resolve().parents[1] / "holocron_b200" / "csrc" / "build"
UNITS = ["conv_fprop", "conv_rows", "conv_wgrad", "conv_wgrad_rows", "attention", "pooling", "involution",
         "lambda_layer"]
SERIALISED = re.compile(r"\((C7511|C7519|C7520)\)")
SPILLS = re.compile(r"(\d+) bytes spill stores, (\d+) bytes spill loads")


@pytest.mark.parametrize("unit", UNITS)
def test_no_serialised_wgmma(unit):
    log = BUILD / f"{unit}.log"
    if not log.exists():
        pytest.skip(f"{log.name} absent: build the library first (python -m holocron_b200.csrc.build)")
    text = log.read_text()
    assert "Compiling entry function" in text, f"{log.name} holds no ptxas -v output"
    notes = [line.strip()[:160] for line in text.splitlines() if SERIALISED.search(line)]
    assert not notes, f"{unit}: {len(notes)} wgmma serialisation note(s), first: {notes[0]}"
    spills = [m.group(0) for m in SPILLS.finditer(text) if m.group(1) != "0" or m.group(2) != "0"]
    assert not spills, f"{unit}: register spills: {spills}"
