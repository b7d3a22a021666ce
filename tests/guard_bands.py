"""Guard-banded calls: does a kernel read and write only its own operands?

Each operand sits inside a larger byte buffer, behind and ahead of guard bands of GUARD bytes, and `guarded_call` runs
the call three times on the same inputs: on plain torch tensors, and twice on guarded buffers with different fills:
  run A: output regions and their guards hold one byte pattern; the guards around the inputs hold NaN (fp16 0x7E00,
         bf16 0x7FC0, int16 weights 0x7F7F, int8 codes and other integers 0x7F, fp32 0x7FC00000);
  run B: a second output pattern; the guards around the inputs hold zeros.
After each guarded run every guard byte, and every byte of a read-only operand, must be unchanged (out-of-bounds or
stray stores), and the outputs of A, B and the plain run must be bit-identical: an element a kernel forgets to write
keeps its fill and differs between A and B, and a read past an input feeds NaN in one run and zero in the other."""
import ctypes

import numpy as np
import torch

DEV = "cuda:0"
GUARD = 4096          # bytes of guard before and after every operand: more than any tile row or vector access here
OUT_FILL = (0xA5, 0x5A)
_NAN = {torch.float16: (torch.int16, 0x7E00), torch.bfloat16: (torch.int16, 0x7FC0), torch.int16: (torch.int16, 0x7F7F),
        torch.float32: (torch.int32, 0x7FC00000)}


class Op:
    """One operand of a call.  kind: "in" (read only, must stay unchanged), "io" (updated in place, compared), "out"
    (written, compared), "scratch" (workspace the call writes before it reads: pattern-filled, not compared), "zeroed"
    (workspace that must be zero before the call: zero-filled, not compared).  `offset` moves the operand that many
    bytes past a 16-byte boundary."""

    def __init__(self, kind, t=None, shape=None, dtype=None, offset=0):
        self.kind, self.t, self.offset = kind, t, offset
        self.shape = tuple(t.shape) if t is not None else tuple(shape)
        self.dtype = t.dtype if t is not None else dtype
        self.nbytes = int(np.prod(self.shape)) * torch.empty(0, dtype=self.dtype).element_size()


def _guard_fill(buf, op, run):
    if op.kind in ("in", "io") and run == 0:
        if op.dtype in _NAN:
            it, pat = _NAN[op.dtype]
            buf.view(it).fill_(pat)
        else:
            buf.fill_(0x7F)
    elif op.kind in ("in", "io"):
        buf.zero_()
    else:
        buf.fill_(OUT_FILL[run])


def _place(op, run, device):
    start = GUARD + op.offset
    total = -(-(start + op.nbytes + GUARD) // 16) * 16
    buf = torch.empty(total, dtype=torch.uint8, device=device)
    _guard_fill(buf, op, run)
    region = buf[start:start + op.nbytes]
    view = region.view(op.dtype).view(op.shape)
    if op.kind in ("in", "io"):
        view.copy_(op.t)
    elif op.kind == "zeroed":
        region.zero_()
    return buf, view, start


def _plain(op, device):
    if op.kind in ("in", "io"):
        return op.t.clone().to(device)
    if op.kind == "zeroed":
        return torch.zeros(op.shape, dtype=op.dtype, device=device)
    return torch.empty(op.shape, dtype=op.dtype, device=device)


def _bytes(t):
    return t.contiguous().view(-1).view(torch.uint8).clone()


def _sync(device):
    if torch.device(device).type == "cuda":
        torch.cuda.synchronize()


def guarded_call(call, ops, device=DEV):
    """Runs call(views) in guarded runs A and B and on plain tensors (see the module docstring); returns the plain run's
    outputs.  call returns the entry's return code, which must be 0."""
    outs = []
    for run in (0, 1):
        placed = {name: _place(op, run, device) for name, op in ops.items()}
        before = {name: p[0].clone() for name, p in placed.items()}
        rc = call({name: p[1] for name, p in placed.items()})
        assert rc == 0, rc
        _sync(device)
        for name, (buf, view, start) in placed.items():
            end = start + ops[name].nbytes
            assert torch.equal(buf[:start], before[name][:start]), f"{name}: guard before the operand written (run {'AB'[run]})"
            assert torch.equal(buf[end:], before[name][end:]), f"{name}: guard after the operand written (run {'AB'[run]})"
            if ops[name].kind == "in":
                assert torch.equal(buf, before[name]), f"{name}: read-only operand written (run {'AB'[run]})"
        outs.append({name: _bytes(placed[name][1]) for name, op in ops.items() if op.kind in ("io", "out")})
    for name in outs[0]:
        assert torch.equal(outs[0][name], outs[1][name]), f"{name}: output differs between fills A and B"
    plain = {name: _plain(op, device) for name, op in ops.items()}
    assert call(plain) == 0
    _sync(device)
    for name in outs[0]:
        assert torch.equal(outs[0][name], _bytes(plain[name])), f"{name}: guarded output differs from the plain call"
    return plain


def _st():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _p(t):
    return t.data_ptr()


def _code(dtype):
    return 0 if dtype == torch.float16 else 1
