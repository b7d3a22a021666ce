"""Host-side mirror of the reference's quantized linear module.

Same names, constructor / classmethod signatures, buffer names, shapes and dtypes, and
the same dispatch rule as awq/quantize/qmodule.py (WQLinear :78-235, pack_intweight
:26-65, calculate_zeros_width :11-23), so state dicts (`qweight`, `scales`,
`scaled_zeros`, `bias`) are interchangeable and the parity tests read like the
reference's call sites.  The packer is a closed-form, vectorised restatement (no
per-column Python loop); the forward pass calls the sm_90a kernels through the
`awq_inference_engine` extension and nothing else — there is no CPU or PyTorch fallback.
"""
import torch
import torch.nn as nn

from .engine import engine as _get_engine


def make_divisible(c, divisor):
    return (c + divisor - 1) // divisor


def calculate_zeros_width(in_features, group_size=128, pack_num=8):
    """Number of 8-row blocks in `scales` / `scaled_zeros` (reference qmodule.py:11-23)."""
    if group_size >= 128:
        size_multiplier = 1
    elif group_size == 64:
        size_multiplier = 2
    elif group_size == 32:
        size_multiplier = 4
    else:
        raise NotImplementedError
    base_width = make_divisible(in_features // group_size, pack_num)
    return make_divisible(base_width, size_multiplier) * size_multiplier


def _packed_coords(N, K, device):
    """(row, int16 column, nibble) of every (n, k) in the packed tensor.

    In the 16-byte chunk of (row n, 32-k block), viewed as four uint32 `u`, nibble `i` of
    word `u` holds k_local = 8*(i % 4) + 2*u + i // 4; chunks are laid out
    [4 rows] x [2 k-blocks] inside one 128-byte segment per (4 rows, 64 k)."""
    n = torch.arange(N, device=device).view(N, 1)
    k = torch.arange(K, device=device).view(1, K)
    o = k % 32
    u = (o >> 1) & 3
    i = (o >> 3) + 4 * (o & 1)
    col = (k // 64) * 64 + (n % 4) * 16 + ((k % 64) // 32) * 8 + u * 2 + i // 4
    return (n // 4).expand(N, K), col.expand(N, K), (i % 4).expand(N, K)


def pack_intweight(unpacked_qweight, interleave=4, kstride=64):
    """[N, K] integers -> int16 [N // 4, K] (reference qmodule.py:26-65).

    Like the reference, the four values of one int16 are OR-ed together UNMASKED
    (qmodule.py:50-55): integers outside 0..15 spill into the neighbouring nibbles exactly
    as they do there (from_linear on weights that were not fake-quantised first)."""
    assert interleave == 4 and kstride == 64, "only the reference's (4, 64) interleave exists"
    q = unpacked_qweight.to(torch.int32)
    N, K = q.shape
    assert N % 4 == 0 and K % 64 == 0
    # P[r, 64*tile + 16*row + 8*blk + 2*u + hi] nibble j  <-  q[4r + row, 64*tile + 32*blk + 8*j + 2*u + hi]
    v = q.view(N // 4, 4, K // 64, 2, 4, 4, 2).permute(0, 2, 1, 3, 5, 6, 4).reshape(N // 4, K, 4)
    out = v[..., 0] | (v[..., 1] << 4) | (v[..., 2] << 8) | (v[..., 3] << 12)
    out = ((out + 32768) & 0xFFFF) - 32768        # numpy astype("int16") wrap-around (qmodule.py:59)
    return out.to(torch.int16).contiguous()


def unpack_intweight(qweight):
    """int16 [N // 4, K] -> uint8 [N, K] of nibbles 0..15 (inverse of pack_intweight)."""
    R, K = qweight.shape
    r, c, j = _packed_coords(R * 4, K, qweight.device)
    p = qweight.to(torch.int32) & 0xFFFF
    return ((p[r, c] >> (4 * j)) & 0xF).to(torch.uint8)


class WQLinear(nn.Module):
    """Drop-in for awq.quantize.qmodule.WQLinear (reference qmodule.py:78-235)."""

    def __init__(self, w_bit, group_size, in_features, out_features, bias, dev, dtype=torch.float16):
        super().__init__()
        if w_bit not in [4]:
            raise NotImplementedError("Only 4-bit are supported for now.")
        self.in_features = in_features
        self.out_features = out_features
        self.w_bit = w_bit
        self.group_size = group_size if group_size != -1 else in_features
        self.split_k_iters = 8  # kept for state/attribute compatibility; unused by these kernels
        self.interleave = 4
        assert self.in_features % self.group_size == 0
        assert out_features % (32 // self.w_bit) == 0
        assert out_features % self.interleave == 0
        pack_num = 32 // self.w_bit
        int16_pack_num = 16 // self.w_bit
        rows = calculate_zeros_width(in_features, self.group_size) * pack_num
        self.register_buffer(
            "qweight",
            torch.zeros((out_features // self.interleave, in_features // int16_pack_num * self.interleave),
                        dtype=torch.int16, device=dev))
        self.register_buffer("scales", torch.zeros((rows, out_features), dtype=dtype, device=dev))
        self.register_buffer("scaled_zeros", torch.zeros((rows, out_features), dtype=dtype, device=dev))
        if bias:
            self.register_buffer("bias", torch.zeros((out_features), dtype=dtype, device=dev))
        else:
            self.bias = None

    @classmethod
    def from_linear(cls, linear, w_bit, group_size, init_only=False, scales=None, zeros=None):
        """Quantise-and-pack an nn.Linear given per-(row, group) scales / integer zeros.

        Restates reference qmodule.py:139-199 without the per-input-channel Python loop;
        element-wise arithmetic is done in the layer's dtype exactly like the reference."""
        awq_linear = cls(w_bit, group_size, linear.in_features, linear.out_features, linear.bias is not None,
                         linear.weight.device, dtype=linear.weight.data.dtype)
        if init_only:
            return awq_linear
        assert scales is not None and zeros is not None
        G = awq_linear.group_size
        dtype = scales.dtype
        ng = scales.shape[1]
        rows = awq_linear.scales.shape[0]
        scale_zeros = zeros * scales
        qscales = torch.zeros((scales.shape[0], rows), dtype=dtype, device=scales.device)
        qscales[:, :ng] = scales
        awq_linear.scales = qscales.transpose(1, 0).contiguous()
        if linear.bias is not None:
            awq_linear.bias = linear.bias.clone().to(dtype)
        w = linear.weight.data
        intweight = torch.round((w + scale_zeros.repeat_interleave(G, dim=1))
                                / scales.repeat_interleave(G, dim=1)).to(torch.int32)
        awq_linear.qweight = pack_intweight(intweight.contiguous(), interleave=4, kstride=64)
        scaled_zeros = torch.zeros_like(qscales)
        scaled_zeros[:, :ng] = -(qscales[:, :ng] * zeros.to(torch.int32).to(torch.float32)).to(dtype)
        awq_linear.scaled_zeros = scaled_zeros.transpose(1, 0).contiguous()
        return awq_linear

    @torch.no_grad()
    def forward(self, x, residual=None):
        """x W~^T (+ bias) (+ residual).  With a bias or a residual, one launch adds them in the kernel's epilogue,
        bit-identical to the reference's `out + self.bias` and the decoder block's `residual + out`."""
        eng = _get_engine()
        inputs = x if x.is_contiguous() else x.contiguous()
        if self.bias is not None or residual is not None:
            return eng.w4a16_linear_forward_cuda(inputs, self.qweight, self.scales, self.scaled_zeros, self.group_size,
                                                 bias=self.bias, residual=residual)
        m = inputs.numel() // inputs.shape[-1]
        if inputs.numel() / inputs.shape[-1] < 8:  # reference dispatch rule, qmodule.py:206
            out = eng.gemv_forward_cuda_new(inputs, self.qweight, self.scales, self.scaled_zeros,
                                            m, self.out_features, self.in_features, self.group_size)
        else:
            out = eng.gemm_forward_cuda_new(inputs, self.qweight, self.scales, self.scaled_zeros)
        return out + self.bias if self.bias is not None else out

    @torch.no_grad()
    def norm_forward(self, x, norm):
        """RMSNorm(x) W~^T (+ bias) with norm = (weight, eps), the decoder's RMSNorm in front of this projection
        (`input_layernorm` before q/k/v); norm=None is forward(x).  Bit-identical to `layernorm_forward_cuda` followed
        by forward(); one fp16 token (and up to 4 tokens, or one bf16 token) normalises inside the W4A16 launch.
        (A method of its own rather than a `norm` argument of forward(): forward's parameters (x, residual) are part
        of this module's tested interface.  There is no norm + residual route.)"""
        if norm is None:
            return self.forward(x)
        weight, eps = norm
        inputs = x if x.is_contiguous() else x.contiguous()
        return _get_engine().rmsnorm_w4a16_linear_forward_cuda(inputs, weight, float(eps), self.qweight, self.scales,
                                                               self.scaled_zeros, self.group_size, bias=self.bias)

    def extra_repr(self) -> str:
        return "in_features={}, out_features={}, bias={}, w_bit={}, group_size={}".format(
            self.in_features, self.out_features, self.bias is not None, self.w_bit, self.group_size)
