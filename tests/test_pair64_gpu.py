"""GEMMs requested with force_bn 2064 (the 256 x 64 CTA-pair tile width of other architectures; on sm_90a the 128 x 64
kernel): the same op-level parity bodies as tests/test_ops_gpu.py."""
import pytest
import torch

import test_ops_gpu as ops

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def L():
    from spann3r_b200 import _lib
    _lib.require_device()
    return _lib


@pytest.mark.parametrize("rows,K,N,groups", [(768, 768, 768, 2), (768, 3072, 768, 2), (768, 1024, 1024, 1), (768, 4096, 1024, 1),
                                             (1536, 768, 96, 1), (512, 96, 1536, 1)])      # even m-tile counts only
def test_pair64_linear(L, rows, K, N, groups):
    ops.test_linear_bias_gelu_residual(L, rows, K, N, groups, 2064)


@pytest.mark.parametrize("rows,C,N,groups,swap", [(768, 768, 768, 2, 1), (768, 768, 2304, 2, 0), (1024, 768, 768, 1, 0)])
def test_pair64_folded_layernorm_chain(L, rows, C, N, groups, swap):
    ops.test_folded_layernorm_chain(L, rows, C, N, groups, swap, 2064)


def test_pair64_conv3x3(L):
    ops.test_conv3x3(L, 1, 24, 32, 96, 256, 1, 2064)
    ops.test_conv3x3(L, 1, 96, 128, 256, 128, 2, 2064)
