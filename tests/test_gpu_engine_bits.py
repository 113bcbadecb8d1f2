"""The wgmma GEMM engine computes the same bits as when tests/golden/engine_bits.json was written: plain and odd-sized
kfac_gemm_tn_tc calls, one grouped launch with every feature, the factor SYRK with and without split partials, a
full ResNet-50 kfac_eigh_batched call and one kfac_precondition call (cases in gen_engine_bits.py)."""
import json

import pytest

import gen_engine_bits as G

pytestmark = pytest.mark.gpu

with open(G.GOLDEN) as _f:
    DIGESTS = json.load(_f)['digests']


@pytest.mark.parametrize('name', sorted(G.CASES))
def test_engine_bits(name):
    assert G.CASES[name]() == DIGESTS[name]
