"""The wgmma GEMM engine computes the same bits as when tests/golden/engine_bits.json was written: plain and odd-sized
kfac_gemm_tn_tc calls, one grouped launch with every feature, the factor SYRK with and without split partials, a
full ResNet-50 kfac_eigh_batched call and kfac_precondition calls over every item kind and method (cases in
gen_engine_bits.py), each with the number of kernel launches it made."""
import json

import pytest

import gen_engine_bits as G

pytestmark = pytest.mark.gpu

with open(G.GOLDEN) as _f:
    _GOLDEN = json.load(_f)
DIGESTS, LAUNCHES = _GOLDEN['digests'], _GOLDEN['launches']


@pytest.mark.parametrize('name', sorted(G.CASES))
def test_engine_bits(name):
    assert G.run(name) == (DIGESTS[name], LAUNCHES[name])
