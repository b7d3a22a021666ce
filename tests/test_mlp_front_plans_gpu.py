"""The MLP front half (b200awq_w4a16_mlp_front: silu(x Wgate~^T) * (x Wup~^T)) at every plan it reaches on this device,
at the partition edges its SM count puts in the shapes (w4a16_plans.mlp_front_cases).

* The profiler pins each case's launches (tests/kernel_trace.py): the kernels in stream order, their grids and their
  shared memory equal what w4a16_plans.mlp_front_plan() derives from the shape and the SM count.  The fused one-token
  kernel is told apart from the plain decode kernel by its template arguments, w4a16_decode_kernel<true, false>.
* Fused cases (one fp16 token): the kernel sums each product in the plain decode kernel's order and rounds like
  silu_mul_kernel, so y equals b200awq_w4a16_gemv(gate) | b200awq_w4a16_gemv(up) -> b200awq_silu_and_mul bit for bit
  (the mirror confirms that the plain plan has the same split and partition), on a probe token and on a randn token
  whose products stay in the range where the SiLU line's roundings show.  Both GEMV products are within the
  elementwise bound of test_token_isolation_gpu.py on the plan's edge channels.
* Composed cases: both products are read back from the workspace, each within the bound on the plan's edge tokens and
  channels; y equals b200awq_silu_and_mul on them bit for bit; where the projection's plan is the GEMV or GEMM entry's,
  each product equals that entry's output bit for bit.
* y and the workspace start as NaN, so an element no CTA stores fails.  Inputs are AWQ-like probe tokens.
* The plugin's retry with a workspace on a shape the fused kernel declines, and QuantLlamaMLP's
  legacy_gemm_zero_offset branch, against the C entry."""
import ctypes
import re

import numpy as np
import pytest
import torch

import llm_awq_b200 as P
from awq_testutil import gen_layer
from kernel_trace import short_names, trace
from oracle import w4a16_oracle as O
from test_token_isolation_gpu import bound_violations, gamma, oracle_terms, probe_tokens, run
from w4a16_plans import edge_channels, edge_tokens, mlp_front_cases, mlp_front_plan, plan

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
DTYPE = {"f16": torch.float16, "bf16": torch.bfloat16}
ERR_WORKSPACE = -6
# the SM count decides every case; without a device the cases are only collected (and skipped), for an H100 SXM
SMS = torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else 132
CASES = mlp_front_cases(SMS)
FUSED = [c for c in CASES if dict(c.expect)["route"] == "fused"]
COMPOSED = [c for c in CASES if dict(c.expect)["route"] != "fused"]


def _p(t):
    return ctypes.c_void_p(t.data_ptr())


def _st():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def mlp_front(x, gate, up, workspace=True):
    """(rc, y, workspace as [2, m, n] of T or None) of b200awq_w4a16_mlp_front; y and the workspace NaN-filled."""
    m, k = x.shape
    n = gate[1].shape[1]
    y = torch.full((m, n), float("nan"), dtype=x.dtype, device=DEV)
    ws = torch.full((2, m, n), float("nan"), dtype=x.dtype, device=DEV) if workspace else None
    nb = P.lib().b200awq_w4a16_mlp_front_workspace_bytes(m, n, k) if workspace else 0
    assert not workspace or nb == ws.numel() * 2
    rc = P.lib().b200awq_w4a16_mlp_front(_p(x), *map(_p, gate), *map(_p, up), _p(y), m, n, k, 128,
                                         0 if x.dtype == torch.float16 else 1, _p(ws) if workspace else None, nb, _st())
    return rc, y, ws


def silu_and_mul(g, u):
    """b200awq_silu_and_mul on the rows [g | u]."""
    m, n = g.shape
    xin = torch.cat([g, u], dim=1).contiguous()
    y = torch.full((m, n), float("nan"), dtype=g.dtype, device=DEV)
    rc = P.lib().b200awq_silu_and_mul(_p(xin), _p(y), m, n, 0 if g.dtype == torch.float16 else 1, _st())
    assert rc == 0, P.lib().b200awq_strerror(rc)
    return y


def assert_bit_identical(got, want, what):
    a, b = got.view(torch.int16), want.view(torch.int16)
    if not torch.equal(a, b):
        bad = (a != b).nonzero()
        i = tuple(bad[0].tolist())
        pytest.fail(f"{what}: {len(bad)} of {a.numel()} elements differ; first at {i}: {got[i].item()!r} against "
                    f"{want[i].item()!r}")


def assert_within_bound(y, x, layer, p, what):
    """The plan's edge tokens and channels of the product y = x W~^T within the elementwise bound."""
    m, n = y.shape
    T = y.dtype
    toks, cols = edge_tokens(p, m), edge_channels(p, n)
    Y, A, D = oracle_terms(x[toks], *layer, T, cols=cols)
    got = y[toks][:, cols].double().cpu().numpy()
    bad = bound_violations(got, Y, A, D, T, gamma(p.route, T), digits=p.route == "decode")
    if bad.any():
        i, j = np.argwhere(bad)[0]
        pytest.fail(f"{what}: {int(bad.sum())} of {bad.size} sampled elements outside the bound; first: token "
                    f"{toks[i]}, channel {cols[j]}: y = {got[i, j]!r}, oracle = {Y[i, j]!r}, A = {A[i, j]!r}; plan {p}")


def layers(c):
    T = DTYPE[c.dtype]
    return gen_layer(c.n, c.k, T, seed=c.n + 3 * c.k, device=DEV), gen_layer(c.n, c.k, T, seed=c.n + 3 * c.k + 1, device=DEV)


def tokens(c):
    x = probe_tokens(c.m, c.k, seed=c.m * 7 + c.k).to(DTYPE[c.dtype])
    return x, x.to(DEV)


# ------------------------------------------------------------------------------------------------ plans pinned
def launch_name(name):
    """The short name of a kernel in the trace: the fused decode instantiation keeps its template arguments."""
    if re.search(r"w4a16_decode_kernel<\s*true\s*,\s*false\s*>", name):
        return "w4a16_decode_kernel<true, false>"
    if "silu_mul_kernel" in name:
        return "silu_mul_kernel"
    found = short_names([name])
    return found.pop() if found else name


def traced_call(i):
    """kernel_trace builder: b200awq_w4a16_mlp_front of CASES[i] on zero weights, with a workspace."""
    c = CASES[i]
    T = DTYPE[c.dtype]
    x, y = torch.zeros(c.m, c.k, dtype=T, device=DEV), torch.empty(c.m, c.n, dtype=T, device=DEV)
    gate, up = ((torch.zeros(c.n // 4, c.k, dtype=torch.int16, device=DEV),
                 *(torch.zeros(O.scale_rows(c.k), c.n, dtype=T, device=DEV) for _ in range(2))) for _ in range(2))
    nb = P.lib().b200awq_w4a16_mlp_front_workspace_bytes(c.m, c.n, c.k)
    ws = torch.empty(nb, dtype=torch.uint8, device=DEV)
    st = _st()
    return lambda: P.lib().b200awq_w4a16_mlp_front(_p(x), *map(_p, gate), *map(_p, up), _p(y), c.m, c.n, c.k, 128,
                                                   int(c.dtype == "bf16"), _p(ws), nb, st)


def test_launches_pinned_by_profiler():
    name = torch.cuda.get_device_name(0)
    records = trace("test_mlp_front_plans_gpu:traced_call", [[i] for i in range(len(CASES))], per_process=64)
    rows, wrong = [], []
    for c, rec in zip(CASES, records):
        ps = mlp_front_plan(c.m, c.n, c.k, c.dtype, SMS)
        # the trace gives static + dynamic shared memory: the stream kernel's 8 bytes of static exchange epochs take
        # one 128-byte unit, the other kernels have none
        want = [(p.kernel, [p.grid, 1, 1], p.smem + (128 if p.route == "stream" else 0)) for p in ps]
        have = [(launch_name(e.name), e.grid, e.smem) for e in rec.events]
        rows.append(f"| {c.id} | {', '.join(h[0] for h in have)} | {[h[1][0] for h in have]} | {[h[2] for h in have]} | "
                    f"{[w[2] for w in want]} |")
        if have != want:
            wrong.append((c.id, have, want))
    print(f"\n{name}, {SMS} SMs\n| case | kernels | grids | shared memory | planned |\n|---|---|---|---|---|\n"
          + "\n".join(rows))
    assert not wrong, wrong


# ------------------------------------------------------------------------------------------------ fused kernel
@pytest.mark.parametrize("case", FUSED, ids=lambda c: c.id)
def test_fused_equals_gemv_gemv_silu_and_mul(case):
    c = case
    (fp,) = mlp_front_plan(c.m, c.n, c.k, c.dtype, SMS)
    pp = plan(1, c.n, c.k, "f16", "gemv", SMS)
    assert fp.route == "fused" and pp.route == "decode" and (pp.S, pp.units) == (fp.S, fp.units), (fp, pp)
    gate, up = layers(c)
    x, xd = tokens(c)
    rc, y, _ = mlp_front(xd, gate, up, workspace=False)   # the fused kernel needs no workspace
    assert rc == 0, P.lib().b200awq_strerror(rc)
    g, u = run("gemv", xd, *gate), run("gemv", xd, *up)
    assert_bit_identical(y, silu_and_mul(g, u), f"{c.id}: fused against gemv | gemv -> silu_and_mul")
    assert_within_bound(g, x, gate, pp, f"{c.id} gate")
    assert_within_bound(u, x, up, pp, f"{c.id} up")
    # the probe tokens' outliers send many products past the range where silu(g) u is finite and non-zero: once more on
    # a randn token, whose products stay where the SiLU line's roundings show
    xr = torch.randn(1, c.k, generator=torch.Generator().manual_seed(c.k)).to(torch.float16).to(DEV)
    rc, y, _ = mlp_front(xr, gate, up, workspace=False)
    assert rc == 0, P.lib().b200awq_strerror(rc)
    g, u = run("gemv", xr, *gate), run("gemv", xr, *up)
    assert torch.isfinite(g).all() and torch.isfinite(u).all()
    assert_bit_identical(y, silu_and_mul(g, u), f"{c.id}: fused against gemv | gemv -> silu_and_mul on a randn token")


# ------------------------------------------------------------------------------------------------ composed path
@pytest.mark.parametrize("case", COMPOSED, ids=lambda c: c.id)
def test_composed_products_within_bound_and_silu_and_mul_exact(case):
    c = case
    ps = mlp_front_plan(c.m, c.n, c.k, c.dtype, SMS)
    assert len(ps) == 3
    p = ps[0]
    gate, up = layers(c)
    x, xd = tokens(c)
    rc, y, ws = mlp_front(xd, gate, up)
    assert rc == 0, P.lib().b200awq_strerror(rc)
    g, u = ws[0], ws[1]
    assert_within_bound(g, x, gate, p, f"{c.id} gate")
    assert_within_bound(u, x, up, p, f"{c.id} up")
    assert_bit_identical(y, silu_and_mul(g, u), f"{c.id}: y against silu_and_mul on the workspace's products")
    same = [e for e in ("gemv", "gemm") if (e == "gemm" or c.m <= 7) and (e == "gemv" or c.n % 128 == 0)
            and plan(c.m, c.n, c.k, c.dtype, e, SMS) == p]
    for e in same:
        assert_bit_identical(g, run(e, xd, *gate), f"{c.id}: gate product against the {e} entry (same plan)")
        assert_bit_identical(u, run(e, xd, *up), f"{c.id}: up product against the {e} entry (same plan)")


# ------------------------------------------------------------------------------------------------ plugin and module
def test_plugin_retries_with_a_workspace_where_the_fused_kernel_declines():
    """One fp16 token on a shape whose fused ring would get fewer than 3 slots: the entry asks for a workspace, and
    mlp_front_forward_cuda calls it again with one; its result is the C entry's composed result."""
    (c,) = [c for c in CASES if c.label == "fused_declines"]
    gate, up = layers(c)
    _, xd = tokens(c)
    rc, _, _ = mlp_front(xd, gate, up, workspace=False)
    assert rc == ERR_WORKSPACE, P.lib().b200awq_strerror(rc)
    rc, want, _ = mlp_front(xd, gate, up)
    assert rc == 0, P.lib().b200awq_strerror(rc)
    got = P.engine().mlp_front_forward_cuda(xd.view(1, 1, c.k), *gate, *up)
    assert got.shape == (1, 1, c.n)
    assert_bit_identical(got.view(1, c.n), want, "mlp_front_forward_cuda against the C entry")


@pytest.mark.parametrize("tokens_", [7, 8, 40])
def test_module_legacy_gemm_zero_offset(tokens_):
    """QuantLlamaMLP(..., legacy_gemm_zero_offset=True) from 8 tokens runs the entry with zeros - 8 scales (the
    reference's GEMM branch); below 8 tokens with the zeros as stored."""
    from llm_awq_b200.fused_mlp import QuantLlamaMLP
    dtype, H, I = torch.float16, 1024, 2816

    def wq(K, N, seed):
        m = P.WQLinear(4, 128, K, N, False, DEV)
        m.qweight, m.scales, m.scaled_zeros = gen_layer(N, K, dtype, seed=seed, device=DEV)
        return m
    gate, up, down = wq(H, I, 41), wq(H, I, 42), wq(I, H, 43)
    mlp = QuantLlamaMLP(gate, down, up, legacy_gemm_zero_offset=True)
    x = probe_tokens(tokens_, H, seed=tokens_).to(dtype).to(DEV)
    got = mlp.our_llama_mlp(x.view(1, tokens_, H))
    off = 8 if tokens_ >= 8 else 0
    rc, want, _ = mlp_front(x, (gate.qweight, gate.scales, gate.scaled_zeros - off * gate.scales),
                            (up.qweight, up.scales, up.scaled_zeros - off * up.scales))
    assert rc == 0, P.lib().b200awq_strerror(rc)
    assert got.shape == (1, tokens_, I)
    assert_bit_identical(got.view(tokens_, I), want, f"QuantLlamaMLP at {tokens_} tokens against the entry")
    if off:   # the offset is applied: the entry with the zeros as stored gives a different result
        _, plain, _ = mlp_front(x, (gate.qweight, gate.scales, gate.scaled_zeros), (up.qweight, up.scales, up.scaled_zeros))
        assert not torch.equal(plain.view(torch.int16), want.view(torch.int16))
