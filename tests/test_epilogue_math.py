"""CPU: the erf approximation the bias + GELU kernels use (vil_epilogue.cuh::gelu_terms, Abramowitz-Stegun 7.1.26) restated
in numpy with the constants PARSED FROM THE CUDA SOURCE, against math.erf: value and derivative of the exact-form GELU
(nn.GELU(), reference Mlp src/models/msvit.py:15-33) must stay within the error the GPU tests assume (fp32 tolerance 2e-6
norm-relative).  Also the grid / slab planning arithmetic of the column-sum launcher, restated from vil_epilogue.cu."""
import math
import os
import re

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = open(os.path.join(ROOT, "vision_longformer_b200", "csrc", "vil_epilogue.cuh")).read()


def _consts():
    body = SRC[SRC.index("gelu_terms(float u)"):SRC.index("__device__ __forceinline__ float gelu_f")]
    nums = [float(x) for x in re.findall(r"(-?\d+\.\d+)f", body)]
    return body, nums


def test_source_constants_are_abramowitz_stegun_7_1_26():
    body, nums = _consts()
    for c in (0.3275911, 1.061405429, -1.453152027, 1.421413741, -0.284496736, 0.254829592, 0.70710678118654752):
        assert any(abs(c - n) < 1e-9 for n in nums), c
    assert any(abs(n + 1.0 / (2.0 * math.log(2.0))) < 1e-12 for n in nums)        # e^{-u^2/2} = 2^{-u^2 / (2 ln 2)}
    assert "ex2_approx" in body and "rcp_approx" in body


def _gelu_terms(u):
    ax = np.abs(u) * 0.70710678118654752
    e = np.exp2(-0.72134752044448170 * u * u)
    t = 1.0 / (0.3275911 * ax + 1.0)
    pl = 1.061405429 * t - 1.453152027
    pl = pl * t + 1.421413741
    pl = pl * t - 0.284496736
    pl = pl * t + 0.254829592
    q = 0.5 * pl * t * e
    return np.where(u >= 0, 1.0 - q, q), e


def test_gelu_value_and_derivative_error():
    u = np.linspace(-9.0, 9.0, 200001)
    phi, gauss = _gelu_terms(u)
    exact_phi = 0.5 * (1.0 + np.vectorize(math.erf)(u / math.sqrt(2.0)))
    assert np.max(np.abs(phi - exact_phi)) < 1e-7                         # 0.5 x the 1.5e-7 bound of A&S 7.1.26
    gelu, gelu_exact = u * phi, u * exact_phi
    grad = phi + u * 0.39894228040143268 * gauss
    grad_exact = exact_phi + u * np.exp(-0.5 * u * u) / math.sqrt(2.0 * math.pi)
    # norm-relative errors on a Gaussian-ish activation distribution (what the GPU tests measure at 2e-6 in fp32)
    w = np.exp(-0.5 * (u / 2.0) ** 2)
    rel = lambda a, b: math.sqrt(np.sum(w * (a - b) ** 2) / np.sum(w * b ** 2))
    assert rel(gelu, gelu_exact) < 2e-7 and rel(grad, grad_exact) < 2e-7
    assert np.max(np.abs(gelu - gelu_exact)) < 6e-7                       # |u| <= 9


def test_column_sum_plan_covers_every_row_and_column():
    """ba_plan (vil_epilogue.cu): column slabs x row slabs must tile the (rows, C) tensor exactly for the widths the nets use."""
    src = open(os.path.join(ROOT, "vision_longformer_b200", "csrc", "vil_epilogue.cu")).read()
    assert "b.ncs = (G + epi::kThreads - 1) / epi::kThreads;" in src and "b.gs = (G + b.ncs - 1) / b.ncs;" in src
    for n in (8, 4):
        for C in (96, 192, 384, 768, 1152, 1536, 3072, 200, 4096):
            if C % n:
                continue
            for rows in (1, 7, 50432, 200960, 803072):
                G = C // n
                ncs = (G + 255) // 256
                gs = (G + ncs - 1) // ncs
                rpi = 256 // gs
                want = (132 * 8) // ncs
                per = max((rows + want - 1) // want, 4 * rpi)
                nrs = max((rows + per - 1) // per, 1)
                assert gs <= 256 and rpi >= 1 and ncs * gs >= G                        # every column group has a thread
                assert nrs * per >= rows and (nrs - 1) * per < rows                    # every row in exactly one slab
