"""bench.py's roofline accounting is pinned to the algorithmic work SURVEY.md section 8(d) computed for the BASELINE
configs (per image, per layer, forward) - the `roofline.achieved` figure is built from these numbers."""
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402

# (nx, ny, w, g, H, M, exact) -> GFLOP per image (SURVEY.md 8(d) "Values [computed]")
SURVEY_GF = [
    ((56, 56, 7, 1, 3, 32, 0), 0.4486), ((56, 56, 7, 1, 3, 32, 1), 0.2384),      # ViL-Small stage 1
    ((28, 28, 7, 1, 3, 64, 0), 0.1856), ((28, 28, 7, 1, 3, 64, 1), 0.1030),      # ViL-Small stage 2
    ((96, 96, 8, 1, 3, 32, 0), 1.825), ((48, 48, 12, 1, 3, 64, 0), 1.596),        # Medium-Deep 384
    ((128, 128, 7, 1, 3, 32, 0), 2.57), ((128, 128, 15, 1, 3, 32, 0), 10.61), ((128, 128, 31, 1, 3, 32, 0), 37.45),
    ((64, 64, 7, 1, 3, 64, 0), 1.19), ((64, 64, 15, 1, 3, 64, 0), 4.38), ((64, 64, 31, 1, 3, 64, 0), 12.12),
]


@pytest.mark.parametrize("args,gf", SURVEY_GF, ids=lambda v: str(v))
def test_flops_match_survey(args, gf):
    nx, ny, w, g, H, M, exact = args
    flops, _ = bench.algorithmic_work(nx, ny, w, g, H, M, exact=exact)
    assert flops / 1e9 == pytest.approx(gf, rel=5e-3)      # SURVEY quotes 3-4 significant digits


def test_bytes_match_survey():
    # SURVEY.md: S1 2.41 MB (+ LSE) and S2 1.21 MB per image forward; all three hot layers 4.82 MB (rounded)
    _, b1 = bench.algorithmic_work(56, 56, 7, 1, 3, 32)
    _, b2 = bench.algorithmic_work(28, 28, 7, 1, 3, 64)
    assert b1 / 1e6 == pytest.approx(2.41, rel=2e-2)
    assert b2 / 1e6 == pytest.approx(1.21, rel=2e-2)
