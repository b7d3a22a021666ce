"""GPU parity of the decode-step attention (`single_query_attention`) at every grouped-query ratio G = H / Hkv and every
head size that is a multiple of 8 up to 256: the ratios of Qwen2 (NVILA, InternVL3), Llama-3.2 and Falcon's multi-query
attention (G = 3, 5, 6, 7, 12, 71; G > 8 runs as several head groups per KV head) and the head sizes the reference
dispatches beyond 64 / 128 / 256.  Checked against oracle/layer_oracle.py, torch's scaled_dot_product_attention and the
stored outputs of the reference's own kernel (tests/golden/reference_kernels_attention.npz).

Tolerances are those of tests/test_attention_gpu.py: 2e-3 (fp16) / 8e-3 (bf16) normwise."""
import os

import numpy as np
import pytest
import torch

import llm_awq_b200 as P
from oracle import layer_oracle as LO
from awq_testutil import dt_name, np64, rel_err
import attention_gqa_cases as C

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
DTYPES = [pytest.param(torch.float16, id="f16"), pytest.param(torch.bfloat16, id="bf16")]
TOL = {torch.float16: 2e-3, torch.bfloat16: 8e-3}
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_kernels_attention.npz")

# (B, L, t): empty cache, one CTA, split over CTAs, circular wrap (t >= L); batch 2 through the fused-QKV views
CONTEXTS = {"t0": (1, 512, 0), "one_cta": (1, 512, 300), "split": (2, 2304, 2100), "wrap": (2, 256, 700)}


def _key_ok(got, want, dtype):
    """The rotated key: within the bound of tests/test_attention_gpu.py (2e-3 of the largest element) or one ulp of T.
    The fp32 angle (thousands of radians at long contexts) can flip the rounding of an element, and one bf16 ulp
    exceeds that bound for elements near the largest."""
    mant = 10 if dtype == torch.float16 else 7
    ulp = 2.0 ** (np.floor(np.log2(np.maximum(np.abs(want), 2.0 ** -14))) - mant)
    return bool(np.all(np.abs(got - want) <= np.maximum(2e-3 * np.abs(want).max(), ulp)))


def _check(B, H, Hkv, D, L, t, dtype, rot_dim=None, base=C.ROPE_BASE, scale=1.0, neox=True, lps=None):
    """Runs one step through the plugin and checks the output against the oracle and the caches: the step's value bit
    for bit, the rotated key as _key_ok, every other slot untouched."""
    eng = P.engine()
    rot_dim = D if rot_dim is None else rot_dim
    _, q, k, v = C.fused_qkv(B, H, Hkv, D, dtype, seed=B * 1000 + H + D + t, device=DEV)
    kc, vc = C.caches(B, Hkv, D, L, dtype, min(t, L) if lps is None else L, seed=t + D + 1, device=DEV)
    kc64, vc64 = np64(kc), np64(vc)
    lps_t = None if lps is None else torch.tensor(lps, dtype=torch.int32, device=DEV)
    out = eng.single_query_attention(q, k, v, kc, vc, lps_t, None, t, rot_dim, base, scale, neox)
    torch.cuda.synchronize()
    want = LO.single_query_attention(np64(q), np64(k), np64(v), kc64, vc64, t, rot_dim, base, scale, neox, dt_name(dtype),
                                     length_per_sample=lps)
    assert out.shape == (B, H, D)
    err = rel_err(np64(out), want)
    assert err < TOL[dtype], err
    got_kc, got_vc = np64(kc), np64(vc)
    assert np.array_equal(got_vc, vc64)
    for b in range(B):
        slot = (t if lps is None else lps[b]) % L
        assert _key_ok(got_kc[b, :, :, slot], kc64[b, :, :, slot], dtype)
        mask = np.ones(L, dtype=bool)
        mask[slot] = False
        assert np.array_equal(got_kc[b, :, :, mask], kc64[b, :, :, mask])


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("ctx", list(CONTEXTS))
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("G,Hkv", [(3, 2), (5, 2), (6, 2), (7, 2), (12, 2), (71, 1)])
def test_group_ratios_vs_oracle(G, Hkv, D, ctx, dtype):
    B, L, t = CONTEXTS[ctx]
    _check(B, G * Hkv, Hkv, D, L, t, dtype)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("ctx", list(CONTEXTS))
@pytest.mark.parametrize("G", [1, 7])
@pytest.mark.parametrize("D", [48, 80, 96, 112, 160, 192, 224])
def test_head_sizes_vs_oracle(D, G, ctx, dtype):
    """Head sizes whose D / 8 does not divide 256: the spare threads of the P.V stage idle."""
    B, L, t = CONTEXTS[ctx]
    _check(B, 2 * G, 2, D, L, t, dtype)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("H,Hkv,D", [(28, 4, 128), (71, 1, 64), (24, 2, 80)])
def test_length_per_sample_partial_interleaved_rotary(H, Hkv, D, dtype):
    """Per-sample lengths over a full cache (one sample wraps, one splits over CTAs), rotary over half the head,
    interleaved pairs, scale 0.5."""
    _check(3, H, Hkv, D, 2304, 77, dtype, rot_dim=D // 2, base=10000.0, scale=0.5, neox=False, lps=[5, 2100, 2400])


@pytest.mark.parametrize("H,Hkv,D", [(28, 4, 128), (71, 1, 64)], ids=["qwen2_7b", "falcon_7b"])
def test_decode_loop_matches_sdpa(H, Hkv, D):
    """40 decode steps from an empty cache against scaled_dot_product_attention on the SAME rotated keys (read back from
    the cache layout): cache writes of every step feed the later ones."""
    eng = P.engine()
    dtype, B, L = torch.float16, 1, 64
    kc = torch.zeros(B, Hkv, D // 8, L, 8, dtype=dtype, device=DEV)
    vc = torch.zeros(B, Hkv, L, D, dtype=dtype, device=DEV)
    for t in range(40):
        _, q, k, v = C.fused_qkv(B, H, Hkv, D, dtype, seed=t, device=DEV)
        out = eng.single_query_attention(q, k, v, kc, vc, None, None, t, D, 10000.0, 1.0, True)
        keys = kc[:, :, :, :t + 1].permute(0, 1, 3, 2, 4).reshape(B, Hkv, t + 1, D).float()
        vals = vc[:, :, :t + 1].float()
        qr = torch.from_numpy(LO.rope_rotate(np64(q), t, D, 10000.0, 1.0, True, "f16")).float().to(DEV)
        ref = torch.nn.functional.scaled_dot_product_attention(qr.view(B, H, 1, D), keys.repeat_interleave(H // Hkv, 1),
                                                               vals.repeat_interleave(H // Hkv, 1))
        assert rel_err(np64(out), np64(ref.view(B, H, D))) < 2e-3, t


@pytest.mark.parametrize("H,Hkv,D", [(28, 4, 128), (71, 1, 64)], ids=["G7", "G71"])
def test_graph_replay_and_repeated_launches(H, Hkv, D):
    """Split contexts leave every head group's arrival counter at zero: repeated launches and CUDA-graph replays agree
    bit for bit."""
    eng = P.engine()
    dtype, B, L, t = torch.float16, 2, 2048, 2000
    _, q, k, v = C.fused_qkv(B, H, Hkv, D, dtype, seed=11, device=DEV)
    kc, vc = C.caches(B, Hkv, D, L, dtype, t, seed=12, device=DEV)
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        first = eng.single_query_attention(q, k, v, kc, vc, None, None, t, D, 10000.0, 1.0, True).clone()
        for _ in range(3):
            assert torch.equal(eng.single_query_attention(q, k, v, kc, vc, None, None, t, D, 10000.0, 1.0, True), first)
        gr = torch.cuda.CUDAGraph()
        side.synchronize()
        with torch.cuda.graph(gr, stream=side):
            o = eng.single_query_attention(q, k, v, kc, vc, None, None, t, D, 10000.0, 1.0, True)
        for _ in range(3):
            gr.replay()
            side.synchronize()
            assert torch.equal(o, first)


def _from_bits(a, dtype):
    return torch.from_numpy(np.ascontiguousarray(a).view(np.int16)).view(dtype).float().numpy().astype(np.float64)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("case", C.REF_CASES, ids=C.case_id)
def test_vs_reference_kernel_outputs(case, dtype):
    """The reference's own kernel (FasterTransformer's masked MHA, built for sm_90a) on the same inputs."""
    B, H, Hkv, D, L, t = case
    eng = P.engine()
    g = np.load(GOLDEN)
    key = f"{dt_name(dtype)}_{C.case_id(case)}"
    q, k, v, kc, vc = C.ref_case_inputs(case, dtype, DEV)
    out = eng.single_query_attention(q, k, v, kc, vc, None, None, t, D, C.ROPE_BASE, 1.0, True)
    torch.cuda.synchronize()
    err = rel_err(np64(out), _from_bits(g[f"out_{key}"], dtype))
    assert err <= TOL[dtype], err
    assert np.array_equal(np64(vc[:, :, t % L]), _from_bits(g[f"vslot_{key}"], dtype))
    assert _key_ok(np64(kc[:, :, :, t % L]), _from_bits(g[f"kslot_{key}"], dtype), dtype)


@pytest.mark.parametrize("H,Hkv,D", [(10, 4, 64), (8, 2, 60), (8, 2, 264)], ids=["heads_not_multiple", "d_not_8", "d_over_256"])
def test_unsupported_shapes_raise(H, Hkv, D):
    eng = P.engine()
    dtype, B, L = torch.float16, 1, 32
    _, q, k, v = C.fused_qkv(B, H, Hkv, D, dtype, seed=0, device=DEV)
    kc = torch.zeros(B, Hkv, D // 8, L, 8, dtype=dtype, device=DEV)
    vc = torch.zeros(B, Hkv, L, D, dtype=dtype, device=DEV)
    with pytest.raises(RuntimeError):
        eng.single_query_attention(q, k, v, kc, vc, None, None, 3, D, 10000.0, 1.0, True)
