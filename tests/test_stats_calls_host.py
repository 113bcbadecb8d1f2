"""The layer helpers make exactly the native calls recorded in tests/golden/stats_calls.json: every entry point, in
order, with every argument (scales as float32 bits, pointers as buffer and offset, geometry structs field by field),
for the cases of gen_stats_calls.py.  Runs on the CPU without the native library."""
import json

import pytest

import gen_stats_calls as G

with open(G.GOLDEN) as _f:
    DIGESTS = json.load(_f)['digests']


def test_cases_match_golden():
    assert sorted(G.CASES) == sorted(DIGESTS)


@pytest.mark.parametrize('name', sorted(G.CASES))
def test_stats_calls(name):
    assert G.digest(name) == DIGESTS[name]
