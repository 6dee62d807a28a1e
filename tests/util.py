"""Shared helpers for the test-suite (golden loading, error metrics)."""
import glob
import os

import torch

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def attn_cases():
    return sorted(os.path.basename(p)[len("attn_"):-3] for p in glob.glob(os.path.join(GOLDEN, "attn_*.pt")))


def load_attn(name):
    return torch.load(os.path.join(GOLDEN, f"attn_{name}.pt"), weights_only=False)


def load_golden(fname):
    return torch.load(os.path.join(GOLDEN, fname), weights_only=False)


def relerr(a, b):
    """norm-relative error ||a-b||_F / ||b||_F in float64."""
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return ((a - b).norm() / b.norm().clamp_min(1e-300)).item()


def load_state(mod, sd):
    """Load a golden state_dict (stored fp32 / int32) into `mod`, keeping mod's dtypes."""
    own = mod.state_dict()
    conv = {k: v.to(own[k].dtype) for k, v in sd.items()}
    mod.load_state_dict(conv, strict=True)
    return mod


# --------------------------------------------------------------------------- measured-error log
# GPU parity tests record the errors they MEASURE (not only assert): conftest.py dumps the table at session end to the
# file named by the VIL_ERRORS_JSON environment variable.
ERRORS = {}


def record(test, case, **vals):
    ERRORS.setdefault(test, {}).setdefault(str(case), {}).update({k: float(v) for k, v in vals.items()})
