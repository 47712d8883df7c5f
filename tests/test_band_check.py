"""CPU: the vote kernel's guard band (DESIGN.md section 4.1) checked empirically.  tools/band_check.c re-states the fast
cone test of csrc/vote.cu next to the reference predicate and searches boundary-concentrated samples for
disagreements that the band would NOT flag (exit code 1); tools/band_check.c runs the full 1e8-sample search."""
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def band_check(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("band") / "band_check")
    cc = os.environ.get("CC", "gcc")
    flags = ["-O2", "-ffp-contract=off"]
    with open("/proc/cpuinfo") as fh:
        if " fma " in fh.read():
            flags.append("-mfma")
    subprocess.check_call([cc] + flags + [os.path.join(ROOT, "tools", "band_check.c"), "-lm", "-o", exe])
    return exe


@pytest.mark.parametrize("thresh,local", [("0.99", "1"), ("0.999", "1"), ("0.9", "1"), ("0.5", "1"), ("0.99", "0")])
def test_no_unflagged_disagreement(band_check, thresh, local):
    r = subprocess.run([band_check, "3000000", thresh, local], stdout=subprocess.PIPE, text=True, timeout=120)
    assert r.returncode == 0, r.stdout
    mism = int(re.search(r"mismatches=(\d+)", r.stdout).group(1))
    ratio = float(re.search(r"analytic bound .* = ([0-9.]+)", r.stdout).group(1))
    assert mism > 1000            # the sampler really sits on the decision boundary
    assert ratio < 0.8            # worst disagreement stays well inside the analytic bound (band = 1.25 x bound)


@pytest.mark.parametrize("thresh", ["0.99", "0.999", "0.5", "0.05"])
def test_no_disagreement_next_to_pixels(band_check, thresh):
    """Hypotheses within a few ulps of, or on, pixels at integer coordinates 0-15 (0 < |h-c| < 1e-6, the reference's
    norm cut): the refit prefilter never decides one wrongly and a one-pixel vote tile flags every disagreement."""
    r = subprocess.run([band_check, "0", thresh, "1"], stdout=subprocess.PIPE, text=True, timeout=120)
    assert r.returncode == 0, r.stdout
    m = re.search(r"near-pixel sweep: (\d+) tests, (\d+) rejected by the norm cut", r.stdout)
    assert int(m.group(1)) == 256000
    assert int(m.group(2)) > 100000          # the sweep really sits inside the norm cut
