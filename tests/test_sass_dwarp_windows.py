"""CPU: static evidence on the built library's SASS (cuobjdump) for the windowed domain-warp kernel the 8192^2 headline runs
(noise_grid2_kernel<simplex, warp, shape 0, windowed>, DESIGN.md section 4): its 8 octaves are one unrolled body with no counter or branch, the
windowed octaves take no mod 289 (4 floors per cell pair instead of 8: 7 * 4 + 8 over the body), at most one constant load per octave (the window
shifts, indexed by the fBm stage), 12 table look-ups per octave, the reference's unfused arithmetic, and fewer instructions than the reducing body
(164 per octave, pinned by tests/test_sass_octave_body.py). A guard against silently losing them, not a performance test. Skipped when cuobjdump
is not installed."""
import os
import re
import shutil
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="cuobjdump not installed")
def test_windowed_octave_body(tw, tmp_path):
    out = str(tmp_path / "octave.txt")
    subprocess.check_call([sys.executable, os.path.join(ROOT, "tools", "sass_excerpt.py"), out])
    lines = open(out).read().split("\n")
    i = next(k for k, ln in enumerate(lines) if ln.startswith("Windowed kernel"))
    assert "unrolled 8-octave body" in lines[i + 1], lines[i + 1]
    hist = dict((m.group(1), float(m.group(2))) for m in re.finditer(r"([A-Z0-9_]+) ([\d.]+)(?:,|$)", lines[i + 2]))
    assert not {"BRA", "ISETP", "UISETP", "UIADD3", "IADD3", "F2I", "I2F"} & set(hist), hist   # no loop counter, branch or integer addressing
    assert hist.get("LDC", 0) <= 1, hist                                                        # the window shifts
    assert hist.get("LDS", 0) == 12, hist                                                       # 6 hash + 6 gradient look-ups per cell pair
    assert hist.get("FRND", 0) == (7 * 4 + 8) / 8, hist                                         # floors: 4 in the 7 windowed octaves, 8 in the last
    assert hist.get("FMUL", 0) >= 40 and hist.get("FADD", 0) >= 40 and hist.get("FFMA", 0) <= 16, hist
    assert sum(hist.values()) <= 157, hist
