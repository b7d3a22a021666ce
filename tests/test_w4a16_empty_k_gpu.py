"""An in_feats with an empty last dimension (k = 0) is rejected with RuntimeError by every W4A16 wrapper of the
extension, before anything is allocated or launched."""
import math

import pytest
import torch

import llm_awq_b200 as P

pytestmark = pytest.mark.gpu

DEV = "cuda:0"


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("lead", [(1,), (4,), (2, 3)], ids=["m1", "m4", "2x3"])
@pytest.mark.parametrize("wrapper", ["gemv", "gemm", "linear", "mlp_front"])
def test_empty_last_dimension_raises(wrapper, lead, dtype):
    eng = P.engine()
    n = 256
    x = torch.empty(*lead, 0, dtype=dtype, device=DEV)
    qw = torch.empty(n // 4, 0, dtype=torch.int16, device=DEV)
    sz = torch.zeros(1, n, dtype=dtype, device=DEV)
    calls = {
        "gemv": lambda: eng.gemv_forward_cuda_new(x, qw, sz, sz, math.prod(lead), n, 0, 128),
        "gemm": lambda: eng.gemm_forward_cuda_new(x, qw, sz, sz),
        "linear": lambda: eng.w4a16_linear_forward_cuda(x, qw, sz, sz, 128),
        "mlp_front": lambda: eng.mlp_front_forward_cuda(x, qw, sz, sz, qw, sz, sz),
    }
    before = eng.launch_count()
    with pytest.raises(RuntimeError, match="non-empty last dimension"):
        calls[wrapper]()
    torch.cuda.synchronize()
    assert eng.launch_count() == before
