"""Gated-MLP module over the one-call front half (`awq_inference_engine.mlp_front_forward_cuda`).

Mirror of the reference's QuantLlamaMLP (tinychat/modules/fused_mlp.py:11-83): same constructor arguments, same
registered buffers and state-dict keys, same forward = down_proj(our_llama_mlp(x)).  The difference is inside
`our_llama_mlp`: the reference makes two engine calls + F.silu + a multiply (four kernels, the intermediate
[m, inter] tensors written and re-read); here it is one engine call -- for one fp16 token one kernel that reads x
once and streams both weight sets through one shared-memory ring.  The zeros tensors are passed AS STORED on every
branch (the reference's GEMM branch subtracts 8 * scales, :69,76, which is inconsistent with WQLinear.forward and with
its own GEMV branch -- SURVEY.md §8a Q3; callers that want that branch pass `legacy_gemm_zero_offset=True`).
"""
import torch
import torch.nn as nn

from .engine import engine


class QuantLlamaMLP(nn.Module):
    def __init__(self, gate_proj, down_proj, up_proj, legacy_gemm_zero_offset=False):
        super().__init__()
        self.register_buffer("gate_proj_qweight", gate_proj.qweight)
        self.register_buffer("gate_proj_scales", gate_proj.scales)
        self.register_buffer("gate_proj_scaled_zeros", gate_proj.scaled_zeros)
        self.register_buffer("up_proj_qweight", up_proj.qweight)
        self.register_buffer("up_proj_scales", up_proj.scales)
        self.register_buffer("up_proj_scaled_zeros", up_proj.scaled_zeros)
        self.in_features = gate_proj.in_features
        self.intermediate_size = gate_proj.out_features
        self.out_features = down_proj.out_features
        self.w_bit = gate_proj.w_bit
        self.down_proj = down_proj
        self.split_k_iters = down_proj.split_k_iters
        self.legacy_gemm_zero_offset = legacy_gemm_zero_offset

    def forward(self, x, norm=None):
        """down_proj(our_llama_mlp(x)); norm = (weight, eps), the decoder's `post_attention_layernorm` in front of the
        MLP, applied inside the front half's call (our_llama_mlp)."""
        return self.down_proj(self.our_llama_mlp(x, norm))

    def our_llama_mlp(self, x, norm=None):
        """silu(x Wgate~^T) * (x Wup~^T), or the same of RMSNorm(x) with norm = (weight, eps): bit-identical to
        `layernorm_forward_cuda` followed by the call without it; one fp16 token normalises inside the fused kernel."""
        gz, uz = self.gate_proj_scaled_zeros, self.up_proj_scaled_zeros
        if self.legacy_gemm_zero_offset and x.numel() // x.shape[-1] >= 8:   # fused_mlp.py:69,76
            gz, uz = gz - 8 * self.gate_proj_scales, uz - 8 * self.up_proj_scales
        if norm is not None:
            weight, eps = norm
            return engine().rmsnorm_mlp_front_forward_cuda(x, weight, float(eps), self.gate_proj_qweight,
                                                           self.gate_proj_scales, gz, self.up_proj_qweight,
                                                           self.up_proj_scales, uz)
        return engine().mlp_front_forward_cuda(x, self.gate_proj_qweight, self.gate_proj_scales, gz,
                                               self.up_proj_qweight, self.up_proj_scales, uz)


def make_fused_mlp(m, parent_name=""):
    """Replace every LlamaMLP-shaped module (gate_proj / up_proj / down_proj WQLinears) with QuantLlamaMLP
    (reference: tinychat/modules/fused_mlp.py:86-103)."""
    if m.__class__.__name__ in ["LlamaMLP"]:
        return QuantLlamaMLP(m.gate_proj, m.down_proj, m.up_proj)
    for name, child in m.named_children():
        child = make_fused_mlp(child, parent_name=f"{parent_name}.{name}")
        if isinstance(child, QuantLlamaMLP):
            setattr(m, name, child)
    return m
