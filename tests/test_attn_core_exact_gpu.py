"""The eval attention core (`s3r_attention`, csrc/attention.cu) bit for bit, on inputs where it has exactly one correct
fp32 answer (attn_core_exact.py), computed in fp64 on the GPU.

Every case compares the whole output buffers with `torch.equal`: the fp32 output, and the split-bf16 planes against
split_ref of the expected fp32.  Cells the kernel must not write hold a sentinel that must survive, and V^T's padding
columns hold NaN that must not reach an output.  A mismatch is reported per (tile, head) with the first elements' tile,
head, row, column and the role of the row (one key, uniform, fractional, decoy, ...), which separates a premise that
fails on the tensor cores (one-key rows involve no sum, uniform rows the widest) from a defect of the kernel."""
import pytest
import torch

import attn_core_exact as A
from test_attention_core_gpu import run

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not torch.cuda.is_available(), reason="needs an H100")]


@pytest.fixture(scope="module")
def L():
    from spann3r_b200 import _lib
    _lib.require_device()
    return _lib


def check(L, case, f32=True, planes=True, ldo=None, guard=0, extra_pad=0):
    """Runs the case (V^T padded with NaN to a multiple of 4, plus `extra_pad` columns) and compares every buffer."""
    c = A.make(case)
    exp = A.expect(c, "cuda")
    ldo = ldo or case.heads * A.D
    nk_pad = (case.nk + 3) // 4 * 4 + extra_pad
    o, hi, lo = run(L, c["q"], c["k"], c["v"], case.heads, nk_pad=nk_pad, pad_fill=float("nan"), ldo=ldo, f32=f32,
                    planes=planes, guard=guard)
    eo, eh, el = A.expected_buffers(exp, case.heads, ldo, guard)
    if f32:
        A.assert_exact("fp32", o, eo.cuda(), case, c["role"])
    if planes:
        A.assert_exact("hi plane", hi, eh.cuda(), case, c["role"])
        A.assert_exact("lo plane", lo, el.cuda(), case, c["role"])


@pytest.mark.parametrize("case", A.ENGINE, ids=lambda c: c.id)
def test_engine_shapes_are_exact(L, case):
    check(L, case)


@pytest.mark.parametrize("case", A.RAGGED, ids=lambda c: c.id)
def test_ragged_sizes_are_exact(L, case):
    """nq, nk of 1 .. 300 around the 128-row tiles, with ldo > heads 64, a guard row and 8 more NaN columns of V^T."""
    check(L, case, ldo=case.heads * A.D + 6, guard=1, extra_pad=8)


@pytest.mark.parametrize("layout", ["fp32", "planes", "both"])
@pytest.mark.parametrize("case", A.CONFIG, ids=lambda c: c.id)
def test_output_configurations_are_exact(L, case, layout):
    check(L, case, f32=layout != "planes", planes=layout != "fp32", ldo=case.heads * A.D + 6, guard=1, extra_pad=8)
