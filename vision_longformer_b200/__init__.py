"""vision_longformer_b200: an H100-native (sm_90a) drop-in for ONE hot path of
microsoft/vision-longformer - the 2-D sliding-chunk local + global-token attention that
MODEL.VIT.MSVIT.ATTN_TYPE='longformerhand' selects.  See DESIGN.md / INTEGRATION.md."""
from .attention import B200Long2DSCSelfAttention, make_dropin_class, relative_position_index
from .layernorm import B200LayerNorm
from .msvit import ARCHS, MsViT, build_vil, parse_arch
from .ops import vil_attention, vil_attention_raw_backward, vil_attention_raw_forward

__all__ = ["B200LayerNorm", "B200Long2DSCSelfAttention", "make_dropin_class", "relative_position_index", "ARCHS", "MsViT",
           "build_vil", "parse_arch", "vil_attention", "vil_attention_raw_forward", "vil_attention_raw_backward"]
