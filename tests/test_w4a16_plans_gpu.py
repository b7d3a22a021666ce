"""Every W4A16 plan the dispatch reaches on this device, at the partition edges its SM count puts in the shapes
(w4a16_plans.edge_cases), against the float64 oracle element by element.

* The profiler pins each case's plan: the kernel's name, grid and shared memory in its trace (tests/kernel_trace.py)
  equal what w4a16_plans.plan() derives from the shape and the SM count (the shared memory pins the ring depths).
* Each case's output is checked on the channels and tokens that carry the plan's edges (w4a16_plans.edge_channels,
  edge_tokens) with the elementwise bound of test_token_isolation_gpu.py, on AWQ-like probe tokens (outliers, a
  non-zero-mean group, subnormals).  The output buffer starts as NaN, so an element no CTA stores fails.
* Every plan that splits k over a cluster gives bit-identical results on a second launch.
* Every served projection (w4a16_plans.SERVED) at the token counts of the route boundaries, and at one token count
  where the tile launch splits k and its clusters walk several tiles, under the same bound."""
import ctypes

import numpy as np
import pytest
import torch

import llm_awq_b200 as P
from awq_testutil import gen_layer
from kernel_trace import short_names, trace
from oracle import w4a16_oracle as O
from test_token_isolation_gpu import bound_violations, gamma, oracle_terms, probe_tokens, run
from w4a16_plans import edge_cases, edge_channels, edge_tokens, plan, served_shapes

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
DTYPE = {"f16": torch.float16, "bf16": torch.bfloat16}
# the SM count decides every case; without a device the cases are only collected (and skipped), for an H100 SXM
SMS = torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else 132
CASES = edge_cases(SMS)
BOUNDARY_MS = (1, 4, 5, 7, 8, 9, 16, 17)


def check_plan_output(m, n, k, dtype, entry, what, layer=None):
    """Run the shape on probe tokens; the edge channels and tokens of its plan within the elementwise bound; a second
    launch bit-identical where the plan splits k."""
    p = plan(m, n, k, dtype, entry, SMS)
    T = DTYPE[dtype]
    qw, s, z = layer or gen_layer(n, k, T, seed=n + 3 * k, device=DEV)
    x = probe_tokens(m, k, seed=m * 7 + k).to(T)
    xd = x.to(DEV)
    y = run(entry, xd, qw, s, z)
    if p.S > 1:
        y2 = run(entry, xd, qw, s, z)
        assert torch.equal(y.view(torch.int16), y2.view(torch.int16)), f"{what}: split-k plan {p} is not deterministic"
    toks, cols = edge_tokens(p, m), edge_channels(p, n)
    Y, A, D = oracle_terms(x[toks], qw, s, z, T, cols=cols)
    got = y[toks][:, cols].double().cpu().numpy()
    bad = bound_violations(got, Y, A, D, T, gamma(p.route, T), digits=p.route == "decode")
    if bad.any():
        i, j = np.argwhere(bad)[0]
        t, c = toks[i], cols[j]
        tile = (f", 128-channel tile {c // 128}, token tile {t // p.tn}" if p.tn else "")
        pytest.fail(f"{what}: {int(bad.sum())} of {bad.size} sampled elements outside the bound; first: token {t}, "
                    f"channel {c}{tile}: y = {got[i, j]!r}, oracle = {Y[i, j]!r}, A = {A[i, j]!r}; plan {p}")


# ------------------------------------------------------------------------------------------------ plans pinned
def traced_call(i):
    """kernel_trace builder: CASES[i]'s entry on zero operands."""
    c = CASES[i]
    T = DTYPE[c.dtype]
    x, y = torch.zeros(c.m, c.k, dtype=T, device=DEV), torch.empty(c.m, c.n, dtype=T, device=DEV)
    qw = torch.zeros(c.n // 4, c.k, dtype=torch.int16, device=DEV)
    s, z = (torch.zeros(O.scale_rows(c.k), c.n, dtype=T, device=DEV) for _ in range(2))
    args = [t.data_ptr() for t in (x, qw, s, z, y)] + [c.m, c.n, c.k, 128, int(c.dtype == "bf16")]
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    if c.entry == "gemv":
        return lambda: P.lib().b200awq_w4a16_gemv(*args, st)
    return lambda: P.lib().b200awq_w4a16_gemm(*args, None, 0, st)


def test_plans_pinned_by_profiler():
    name = torch.cuda.get_device_name(0)
    records = trace("test_w4a16_plans_gpu:traced_call", [[i] for i in range(len(CASES))], per_process=64)
    rows, wrong = [], []
    for c, rec in zip(CASES, records):
        p = plan(c.m, c.n, c.k, c.dtype, c.entry, SMS)
        got = [(e.name, e.grid, e.smem) for e in rec.events]
        names = short_names(n for n, _, _ in got)
        grids = [g for _, g, _ in got]
        smem = [sm for _, _, sm in got]
        rows.append(f"| {c.id} | {p.klass} | {', '.join(sorted(names))} | {grids} | {smem} | {p.smem} |")
        # the trace gives static + dynamic shared memory: the stream kernel's 8 bytes of static exchange epochs take
        # one 128-byte unit, the other kernels have none
        if len(got) != 1 or names != {p.kernel} or grids[0] != [p.grid, 1, 1] or \
                smem[0] != p.smem + (128 if p.route == "stream" else 0):
            wrong.append((c.id, got, p.kernel, p.grid))
    print(f"\n{name}, {SMS} SMs\n| case | plan class | kernel | grid | shared memory | planned dynamic |\n"
          "|---|---|---|---|---|---|\n" + "\n".join(rows))
    assert not wrong, wrong


# ------------------------------------------------------------------------------------------------ oracle
@pytest.mark.parametrize("case", CASES, ids=lambda c: c.id)
def test_edge_case_within_elementwise_bound(case):
    check_plan_output(case.m, case.n, case.k, case.dtype, case.entry, case.id)


def multi_tile_split_m(n, k):
    """The smallest token count at which the tile launch splits k and its clusters walk >= 3 tiles (else >= 2), or
    None."""
    for need in (3, 2):
        for m in range(9, 4097):
            p = plan(m, n, k, "f16", "gemm", SMS)
            if p.route == "tile" and p.S > 1 and p.tiles_per_cluster >= need:
                return m
    return None


@pytest.mark.parametrize("dtype", ["f16", "bf16"])
@pytest.mark.parametrize("shape", served_shapes(), ids=lambda s: f"{s[0]}-n{s[1]}-k{s[2]}")
def test_served_shape_within_elementwise_bound(shape, dtype):
    name, n, k = shape
    ms = list(BOUNDARY_MS) + [m for m in (multi_tile_split_m(n, k),) if m]
    layer = gen_layer(n, k, DTYPE[dtype], seed=n + 3 * k, device=DEV)
    for m in ms:
        check_plan_output(m, n, k, dtype, "gemv" if m <= 7 else "gemm", f"{name} m={m} {dtype}", layer)
