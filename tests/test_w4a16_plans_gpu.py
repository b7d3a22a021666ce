"""Every W4A16 plan the dispatch reaches on this device, at the partition edges its SM count puts in the shapes
(w4a16_plans.edge_cases), against the float64 oracle element by element.

* The profiler pins each case's plan: the kernel's name, grid and shared memory in the exported trace equal what
  w4a16_plans.plan() derives from the shape and the SM count (the shared memory pins the ring depths).
* Each case's output is checked on the channels and tokens that carry the plan's edges (w4a16_plans.edge_channels,
  edge_tokens) with the elementwise bound of test_token_isolation_gpu.py, on AWQ-like probe tokens (outliers, a
  non-zero-mean group, subnormals).  The output buffer starts as NaN, so an element no CTA stores fails.
* Every plan that splits k over a cluster gives bit-identical results on a second launch.
* Every served projection (w4a16_plans.SERVED) at the token counts of the route boundaries, and at one token count
  where the tile launch splits k and its clusters walk several tiles, under the same bound."""
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import llm_awq_b200 as P
from awq_testutil import gen_layer
from test_linear_epilogue_gpu import short_names
from test_token_isolation_gpu import bound_violations, gamma, oracle_terms, probe_tokens
from w4a16_plans import edge_cases, edge_channels, edge_tokens, plan, served_shapes

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
DTYPE = {"f16": torch.float16, "bf16": torch.bfloat16}
# the SM count decides every case; without a device the cases are only collected (and skipped), for an H100 SXM
SMS = torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else 132
CASES = edge_cases(SMS)
BOUNDARY_MS = (1, 4, 5, 7, 8, 9, 16, 17)


def call(entry, x, qw, s, z):
    """y of b200awq_w4a16_gemv / _gemm, into a NaN-filled buffer."""
    M, K = x.shape
    N = s.shape[1]
    y = torch.full((M, N), float("nan"), dtype=x.dtype, device=DEV)
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    code = 0 if x.dtype == torch.float16 else 1
    L = P.lib()
    if entry == "gemv":
        rc = L.b200awq_w4a16_gemv(x.data_ptr(), qw.data_ptr(), s.data_ptr(), z.data_ptr(), y.data_ptr(), M, N, K, 128, code, st)
    else:
        rc = L.b200awq_w4a16_gemm(x.data_ptr(), qw.data_ptr(), s.data_ptr(), z.data_ptr(), y.data_ptr(), M, N, K, 128, code,
                                  None, 0, st)
    assert rc == 0, L.b200awq_strerror(rc)
    return y


def check_plan_output(m, n, k, dtype, entry, what, layer=None):
    """Run the shape on probe tokens; the edge channels and tokens of its plan within the elementwise bound; a second
    launch bit-identical where the plan splits k."""
    p = plan(m, n, k, dtype, entry, SMS)
    T = DTYPE[dtype]
    qw, s, z = layer or gen_layer(n, k, T, seed=n + 3 * k, device=DEV)
    x = probe_tokens(m, k, seed=m * 7 + k).to(T)
    xd = x.to(DEV)
    y = call(entry, xd, qw, s, z)
    if p.S > 1:
        y2 = call(entry, xd, qw, s, z)
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
# Child process: for each case [m, n, k, dtype, entry], (name, grid, shared memory) of every kernel of one call in launch
# order, read from the exported Chrome trace, after a first call outside the profiled region (module load, descriptors).
# Entry "mlp_front" is b200awq_w4a16_mlp_front with both weight sets and a workspace.
_PROFILE = """
import ctypes, json, os, sys, tempfile
sys.path[:0] = sys.argv[1:3]
import torch
import llm_awq_b200 as P
from oracle import w4a16_oracle as O
L = P.lib()
out = []
for m, n, k, dt, entry in json.loads(sys.argv[3]):
    dtype = torch.float16 if dt == "f16" else torch.bfloat16
    x = torch.zeros(m, k, dtype=dtype, device="cuda")
    qw = torch.zeros(n // 4, k, dtype=torch.int16, device="cuda")
    s = torch.zeros(O.scale_rows(k), n, dtype=dtype, device="cuda")
    z = torch.zeros_like(s)
    y = torch.empty(m, n, dtype=dtype, device="cuda")
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    code = 0 if dt == "f16" else 1
    if entry == "mlp_front":
        qw2, s2, z2 = torch.zeros_like(qw), torch.zeros_like(s), torch.zeros_like(z)
        nb = L.b200awq_w4a16_mlp_front_workspace_bytes(m, n, k)
        ws = torch.empty(nb, dtype=torch.uint8, device="cuda")
        run = lambda: L.b200awq_w4a16_mlp_front(x.data_ptr(), qw.data_ptr(), s.data_ptr(), z.data_ptr(), qw2.data_ptr(), s2.data_ptr(), z2.data_ptr(), y.data_ptr(), m, n, k, 128, code, ws.data_ptr(), nb, st)
    elif entry == "gemv":
        run = lambda: L.b200awq_w4a16_gemv(x.data_ptr(), qw.data_ptr(), s.data_ptr(), z.data_ptr(), y.data_ptr(), m, n, k, 128, code, st)
    else:
        run = lambda: L.b200awq_w4a16_gemm(x.data_ptr(), qw.data_ptr(), s.data_ptr(), z.data_ptr(), y.data_ptr(), m, n, k, 128, code, None, 0, st)
    assert run() == 0
    torch.cuda.synchronize()
    for attempt in range(3):  # a session that recorded no kernel at all lost its activity records: profile again
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            assert run() == 0
            torch.cuda.synchronize()
        fd, path = tempfile.mkstemp(suffix=".json")
        os.close(fd)
        try:
            prof.export_chrome_trace(path)
            with open(path) as f:
                events = json.load(f)["traceEvents"]
        finally:
            os.unlink(path)
        kernels = [[e["name"], e.get("args", {}).get("grid"), e.get("args", {}).get("shared memory")]
                   for e in sorted((e for e in events if e.get("cat") == "kernel"), key=lambda e: e.get("ts", 0))]
        if kernels:
            break
    out.append(kernels)
print(json.dumps(out))
"""


def profiled_launches(cases, per_process=64):
    tests = os.path.dirname(os.path.abspath(__file__))
    rows = [[c.m, c.n, c.k, c.dtype, c.entry] for c in cases]
    out = []
    for i in range(0, len(rows), per_process):
        r = subprocess.run([sys.executable, "-s", "-c", _PROFILE, os.path.dirname(tests), tests,
                            json.dumps(rows[i:i + per_process])], capture_output=True, text=True, timeout=900)
        assert r.returncode == 0, r.stderr[-3000:]
        out += json.loads(r.stdout.strip().splitlines()[-1])
    return out


def test_plans_pinned_by_profiler():
    name = torch.cuda.get_device_name(0)
    launches = profiled_launches(CASES)
    rows, wrong = [], []
    for c, got in zip(CASES, launches):
        p = plan(c.m, c.n, c.k, c.dtype, c.entry, SMS)
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
