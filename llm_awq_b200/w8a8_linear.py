"""Host-side mirror of the reference's W8A8 linear module (awq/quantize/w8a8_linear.py).

W8A8OF16LinearDynamicInputScale has the reference's constructor and classmethod signatures, buffers (`weight` int8
[OC, IC], `dequant_scale` fp16 [OC]), `bias` attribute (fp16 [OC] or None) and forward dispatch: a layer built with
a bias calls `w8a8_gemm_fuse_bias_forward_cuda`, one without calls `w8a8_gemm_forward_cuda` (w8a8_linear.py:86-137).
The weights are quantised exactly as the reference quantises them (w8a8_linear.py:140-211): per output channel,
s = max|w| clamped at 1e-5 and divided by 127, then round(w / s) -- in the linear's own dtype.  Unlike the reference,
`from_linear` / `from_qkv` do not modify the linear layers they are given, and take a `device` (default: the
current CUDA device, as the reference).  The forward pass runs the sm_90a kernels of `awq_inference_engine`; there
is no PyTorch fallback.
"""
import torch

from .engine import engine as _get_engine


def _default_device(device):
    return torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)


def quantize_weight_per_channel(weight, s1_scale=None):
    """[OC, IC] float weight -> (int8 [OC, IC], fp16 scales [OC]) with the reference's arithmetic
    (w8a8_linear.py:156-166): the division and the rounding happen in the weight's dtype."""
    w = weight.detach().clone()
    if s1_scale is None:
        s1_scale, _ = torch.max(abs(w), dim=-1, keepdim=True)
        s1_scale = s1_scale.clamp_(min=1e-5).div_(127)
    q = w.div_(s1_scale.to(w.device)).round_().to(torch.int8)
    return q, s1_scale.reshape(-1).half()


class W8A8OF16LinearDynamicInputScale(torch.nn.Module):
    """y = (x_q W_q^T) * dequant_scale * input_scale (+ bias), int8 codes in, fp16 out (the reference's
    W8A8OF16LinearDynamicInputScale, awq/quantize/w8a8_linear.py:70-211)."""

    def __init__(self, in_features, out_features, bias=True, scale=1.0, params_dtype=None, device=None):
        super().__init__()
        device = _default_device(device)
        self.in_features = in_features
        self.out_features = out_features
        self.register_buffer("dequant_scale", torch.ones(out_features, dtype=torch.half, device=device))
        self.register_buffer("weight", torch.empty(out_features, in_features, dtype=torch.int8, device=device))
        if bias:
            self.bias = torch.empty(out_features, dtype=torch.float16, device=device)
        else:
            self.register_parameter("bias", None)
        self._fuse_bias = bool(bias)  # the reference picks its apply_weights at construction

    def forward(self, input_, input_scale, output_buffer, residual=None, layer_scale=None):
        """input_ int8 [tokens, IC] codes, input_scale fp16 [tokens], output_buffer fp16 [tokens, OC] (written).

        With `layer_scale` (fp16 [OC]) and / or `residual` (fp16, output_buffer's shape, not sharing its memory),
        output_buffer receives `residual + out * layer_scale` in the GEMM's own launch, bit-identical to the encoder
        layers' PyTorch ops on the plain output (InternViT's `residual + out * self.ls1`, SigLIP's `residual + out`)."""
        e = _get_engine()
        if residual is not None or layer_scale is not None:
            e.w8a8_linear_forward_cuda(input_, self.weight, self.dequant_scale, input_scale, output_buffer,
                                       bias=self.bias if self._fuse_bias else None, layer_scale=layer_scale,
                                       residual=residual)
        elif self._fuse_bias:
            e.w8a8_gemm_fuse_bias_forward_cuda(input_, self.weight, self.dequant_scale, input_scale, output_buffer, self.bias)
        else:
            e.w8a8_gemm_forward_cuda(input_, self.weight, self.dequant_scale, input_scale, output_buffer)

    @classmethod
    def from_linear(cls, linear, init_only=False, s1_scale=None, fc1=False, device=None):
        device = _default_device(device)
        q_linear = cls(linear.in_features, linear.out_features, linear.bias is not None, device=device)
        if init_only:
            return q_linear
        q, s = quantize_weight_per_channel(linear.weight.data, s1_scale)
        if linear.bias is not None:
            q_linear.bias = linear.bias.detach().clone().half().contiguous().to(device)
        q_linear.weight.data[:, :] = q.to(device)
        q_linear.dequant_scale.data[:] = s.to(device)
        return q_linear

    @classmethod
    def from_qkv(cls, q, k, v, init_only=False, s1_scale=None, device=None):
        device = _default_device(device)
        q_linear = cls(q.in_features, q.out_features + k.out_features + v.out_features, q.bias is not None, device=device)
        if init_only:
            return q_linear
        weight = torch.cat([q.weight.data, k.weight.data, v.weight.data], dim=0)
        qw, s = quantize_weight_per_channel(weight, s1_scale)
        if q.bias is not None:
            q_linear.bias = torch.cat([q.bias, k.bias, v.bias], dim=0).detach().half().contiguous().to(device)
        q_linear.weight.data[:, :] = qw.to(device)
        q_linear.dequant_scale.data[:] = s.to(device)
        return q_linear
