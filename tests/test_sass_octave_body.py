"""CPU: static evidence on the built library's SASS (cuobjdump) that the headline kernel runs its 8 octaves as one unrolled body: no counter,
address arithmetic or back-branch per octave, and the instruction count per octave DESIGN.md section 4 quotes. The instruction mix of that
body (unfused arithmetic, table look-ups, no integer addressing) is checked by tests/test_sass_static.py on the same excerpt. A guard against
silently losing the unrolling (a flag change, a compiler update), not a performance test. Skipped when cuobjdump is not installed."""
import os
import re
import shutil
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="cuobjdump not installed")
def test_headline_octave_body_is_unrolled(tw, tmp_path):
    out = str(tmp_path / "octave.txt")
    subprocess.check_call([sys.executable, os.path.join(ROOT, "tools", "sass_excerpt.py"), out])
    lines = open(out).read().split("\n")
    assert "unrolled 8-octave body" in lines[1], lines[1]
    hist = dict((m.group(1), float(m.group(2))) for m in re.finditer(r"([A-Z0-9_]+) ([\d.]+)(?:,|$)", lines[2]))
    assert not {"BRA", "ISETP", "UISETP", "UIADD3", "IADD3", "LDC"} & set(hist), hist   # no loop counter, branch or indexed constant load
    assert sum(hist.values()) <= 164, hist
