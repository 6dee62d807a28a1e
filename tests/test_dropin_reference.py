"""The reference-side binding of INTEGRATION.md section 1 (`make_dropin_class`).

CPU part: the drop-in class built into an MsViT at the seam the reference uses (`AttnBlock.__init__`, msvit.py:269-276)
must reproduce what the reference's own `MsViT` (src/models/msvit.py:343) and `Long2DSCSelfAttention` expose without
running them: state_dict keys and shapes, parameter count, `isinstance` (msvit.py:532-541 `reset_vil_mode`), public
attributes, `compute_macs` (longformer2d.py:231-280), `relative_position_index`.  The reference side is stored in
tests/golden/dropin_reference.pt (oracle/make_golden.py, from the unmodified reference); the base class here is a
stand-in with the reference constructor's signature.

GPU part: the same class factory run forward + backward and compared with the plain module.
"""
import pytest
import torch
from torch import nn

from tests.util import load_golden
from vision_longformer_b200 import B200Long2DSCSelfAttention, MsViT, make_dropin_class


class _StandIn(nn.Module):
    """Same constructor signature as the reference class (longformer2d.py:13-14); used where the reference is absent."""

    def __init__(self, dim, num_heads=8, qkv_bias=False, qk_scale=None, attn_drop=0., proj_drop=0., w=7, d=1,
                 autoregressive=False, sharew=False, nglo=1, only_glo=False, exact=0, autograd=False, rpe=False, mode=0):
        raise AssertionError("the base-class constructor must never run in the drop-in class")


def test_dropin_class_binds_into_reference_msvit():
    gold = load_golden("dropin_reference.pt")
    DropIn = make_dropin_class(_StandIn)
    assert issubclass(DropIn, _StandIn) and issubclass(DropIn, B200Long2DSCSelfAttention)
    torch.manual_seed(0)
    net = MsViT(arch=gold["arch"], img_size=224, num_classes=10, drop_path_rate=0.1, norm_embed=True, sharew=True,
                attn_type="longformerhand", sw_exact=0, mode=1, ln_eps=1e-6, attn_cls=DropIn)
    attn = [m for m in net.modules() if isinstance(m, _StandIn)]
    assert len(attn) == 2 and all(type(m) is DropIn for m in attn)                  # the two s1 stages
    assert all(m.forward.__func__ is B200Long2DSCSelfAttention.forward for m in attn)
    # one parameter set only (the reference constructor must not have run a second time); checkpoints flow both ways
    assert {k: tuple(v.shape) for k, v in net.state_dict().items()} == gold["shapes"]
    assert sum(p.numel() for p in net.parameters()) == gold["n_params"]
    # reset_vil_mode finds the modules through isinstance  (msvit.py:532-541)
    net.reset_vil_mode(0)
    assert all(m.mode == 0 for m in attn)
    net.reset_vil_mode(-1)
    assert all(m.mode == -1 for m in attn)
    # public attributes read elsewhere in the reference
    for a, ref in zip(attn, gold["attrs"]):
        for name, val in ref.items():
            assert getattr(a, name) == val, name
        assert a.query is a.query_global and a.kv is a.kv_global and a.proj is a.proj_global      # sharew
    # the MAC-counting hook gives the reference's number (longformer2d.py:231-280)
    for a, macs in zip(attn, gold["macs_56x56"]):
        x = torch.zeros(1, a.Nglo + 56 * 56, a.num_heads * a.head_dim)
        a.__flops__ = 0
        type(a).compute_macs(a, (x,), None)
        assert a.__flops__ == macs and macs > 0
    # no CPU path: the drop-in class refuses CPU tensors loudly
    with pytest.raises(RuntimeError, match="no CPU"):
        net.eval()(torch.zeros(1, 3, 224, 224))


def test_dropin_nonshared_weights_and_rpe_state_dict():
    gold = load_golden("dropin_reference.pt")
    DropIn = make_dropin_class(_StandIn)
    torch.manual_seed(1)
    mod = DropIn(autograd=False, **gold["rpe_kwargs"])
    assert sorted(mod.state_dict().keys()) == gold["rpe_keys"]
    assert torch.equal(mod.relative_position_index, gold["relative_position_index"])
    assert mod.query is not mod.query_global


def test_dropin_mro_never_runs_the_base_constructor():
    DropIn = make_dropin_class(_StandIn)
    m = DropIn(32, num_heads=2, w=4, nglo=1, sharew=True, rpe=True)
    assert isinstance(m, _StandIn) and isinstance(m, B200Long2DSCSelfAttention)
    assert DropIn.__name__ == "B200_StandIn"
    assert len(list(m.parameters())) == len(list(B200Long2DSCSelfAttention(32, num_heads=2, w=4, nglo=1, sharew=True, rpe=True).parameters()))


@pytest.mark.gpu
def test_dropin_class_runs_on_gpu():
    DropIn = make_dropin_class(_StandIn)
    kw = dict(dim=96, num_heads=3, qkv_bias=True, w=7, nglo=1, sharew=True, rpe=False)
    torch.manual_seed(0)
    a = B200Long2DSCSelfAttention(**kw).cuda().bfloat16()
    b = DropIn(**kw).cuda().bfloat16()
    b.load_state_dict(a.state_dict())
    x = torch.randn(2, 1 + 14 * 14, 96, device="cuda", dtype=torch.bfloat16)
    xa, xb = x.clone().requires_grad_(True), x.clone().requires_grad_(True)
    ya, yb = a(xa, 14, 14), b(xb, 14, 14)
    ya.sum().backward()
    yb.sum().backward()
    assert torch.equal(ya, yb) and torch.equal(xa.grad, xb.grad)
