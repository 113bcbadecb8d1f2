"""Host-only checks of kfac_precondition's planning (no GPU): the workspace it asks for, and how it rejects items.

Every call here is decided before kfac_precondition touches the device: a workspace query, a call without a workspace
(which reports the bytes the call needs under its method), or a call with an item that is malformed or whose
second-order data is missing.  The expected values are in tests/golden/precond_plan.json:

    python tests/test_precond_plan_host.py [OUT.json]     # default: tests/golden/precond_plan.json

The workspace holds one partial-sum slab for every product that splits its reduction (K > 1024).  A product with an
epilogue, or whose output's leading dimension is not the padded width, does not split; the golden values were
written when such products still had a slab, so the expected bytes are the golden ones without those slabs
(unused_slab_bytes)."""
import ctypes as C
import json
import os
import re
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from kfac_b200 import _cabi  # noqa: E402

GOLDEN = os.path.join(HERE, 'golden', 'precond_plan.json')
DENSE, EMB, DIAG_G, TIED, DIAG_A = (_cabi.KFAC_ITEM_DENSE, _cabi.KFAC_ITEM_EMBEDDING, _cabi.KFAC_ITEM_DIAG_G,
                                    _cabi.KFAC_ITEM_TIED, _cabi.KFAC_ITEM_DIAG_A)
KIND_NAMES = {DENSE: 'dense', EMB: 'embedding', DIAG_G: 'diag_g', TIED: 'tied', DIAG_A: 'diag_a'}
METHODS = {'eigen': _cabi.KFAC_EIGEN, 'inverse': _cabi.KFAC_INVERSE}
ld4 = _cabi.ld4
# stand-ins for device pointers: nothing here dereferences them
FAKE = 0x7f0000100000
FAKE_WS = 0x7f0010000000
SIZE_MAX = (1 << 64) - 1


def lib():
    return _cabi.load()


def p_shape(kind, g, a):
    """(rows, columns) of the item's P: the gradient's layout, (V, d) for an embedding or tied item"""
    return (a, g) if kind in (EMB, TIED) else (g, a)


def item(kind, g, a, ldp_pad=0, **fields):
    """A fully ready item with fake pointers: every second-order operand present, leading dimensions padded"""
    it = _cabi.PrecondItem()
    it.kind, it.g, it.a = kind, g, a
    for name in ('wgrad', 'qa', 'qaT', 'qg', 'qgT', 'dgda', 'da', 'dg', 'a_inv', 'g_inv', 'P', 'dh'):
        setattr(it, name, FAKE)
    it.ldqa, it.ldqg, it.ld_dgda = ld4(a), ld4(g), ld4(a)
    it.ldp = ld4(p_shape(kind, g, a)[1]) + ldp_pad
    it.tied_damping = 0.5
    for k, v in fields.items():
        setattr(it, k, v)
    return it


def array(items):
    return (_cabi.PrecondItem * len(items))(*items)


def workspace_bytes(items):
    return lib().kfac_precondition_workspace_bytes(array(items), len(items))


def need(items, method):
    """The bytes kfac_precondition needs under `method`, from its reply to a call without a workspace"""
    L = lib()
    rc = L.kfac_precondition(array(items), len(items), method, 1e-3, None, 0, None)
    assert rc == _cabi.KFAC_ERR_WORKSPACE
    m = re.fullmatch(r'precondition: workspace too small \(0 < (\d+)\)', _cabi.last_error())
    assert m, _cabi.last_error()
    return int(m.group(1))


def slab_bytes(splits, elems):
    return (splits * elems * 4 + 255) // 256 * 256


def unused_slab_bytes(it, method):
    """The slab the workspace once reserved for a last product that does not split: a diagonal item's under the
    inverse method (its product divides in the epilogue), or any item's whose P is not at the padded width"""
    g, a = it.g, it.a
    if it.kind == DENSE:
        n, p_rows, p_ld = g, g, ld4(a)
    elif it.kind == DIAG_A:
        n, p_rows, p_ld = g, g, ld4(a)
    else:
        rows, n = p_shape(it.kind, g, a)
        p_rows, p_ld = rows, ld4(n)
    if n <= 1024:
        return 0
    epilogue = it.kind != DENSE and it.kind != TIED and method == 'inverse'
    if epilogue or it.ldp != p_ld:
        return slab_bytes((n + 511) // 512, p_rows * p_ld)
    return 0


def workspace_corpus():
    """name -> item list: every kind at widths on both sides of the split threshold, with and without padded P"""
    c = {}
    for w in (1023, 1024, 1025, 4100):
        c[f'dense_g{w}'] = [item(DENSE, w, 300)]
        c[f'dense_a{w}'] = [item(DENSE, 300, w)]
        c[f'dense_sq{w}'] = [item(DENSE, w, w)]
        c[f'embedding_d{w}'] = [item(EMB, w, 3000)]
        c[f'diag_g_a{w}'] = [item(DIAG_G, 3000, w)]
        c[f'tied_d{w}'] = [item(TIED, w, 2000)]
        c[f'diag_a_g{w}'] = [item(DIAG_A, w, 3001)]
        c[f'diag_a_a{w}'] = [item(DIAG_A, 300, w)]
    for w in (1023, 1025, 4100):
        for kind, g, a in ((DENSE, w, 300), (DENSE, 300, w), (EMB, w, 3000), (DIAG_G, 3000, w), (TIED, w, 2000),
                           (DIAG_A, w, 3001)):
            c[f'{KIND_NAMES[kind]}_{g}x{a}_ldp_padded'] = [item(kind, g, a, ldp_pad=8)]
    c['all_kinds'] = [item(DENSE, 1100, 1200), item(EMB, 1100, 2000), item(DIAG_G, 1500, 1030), item(TIED, 300, 1000),
                      item(DIAG_A, 1050, 2001), item(DENSE, 64, 65), item(EMB, 64, 100), item(DIAG_G, 100, 9)]
    c['all_kinds_padded'] = [item(DENSE, 1100, 1200, ldp_pad=4), item(EMB, 1100, 2000, ldp_pad=4),
                             item(DIAG_G, 1500, 1030), item(TIED, 300, 1000, ldp_pad=4), item(DIAG_A, 1050, 2001)]
    return c


def not_ready(kind, method):
    """An item of `kind` missing one operand `method` needs, for every operand it needs"""
    vrow = {EMB: 'da', DIAG_G: 'dg', TIED: 'da', DIAG_A: 'da'}
    q = {EMB: 'qg', DIAG_G: 'qa', TIED: 'qg', DIAG_A: 'qg'}
    inv = {EMB: 'g_inv', DIAG_G: 'a_inv', DIAG_A: 'g_inv'}
    if kind == DENSE:
        names = ['qa', 'qaT', 'qg', 'qgT'] if method == 'eigen' else ['a_inv', 'g_inv']
        out = [[n] for n in names]
        if method == 'eigen':
            out += [['dgda', 'da'], ['dgda', 'dg']]
        return out
    if kind == TIED:
        return [['da'], ['qg'], ['qgT'], ['dg'], ['dh']]
    if method == 'eigen':
        return [[vrow[kind]], [q[kind]], [q[kind] + 'T'], [{'da': 'dg', 'dg': 'da'}[vrow[kind]]]]
    return [[vrow[kind]], [inv[kind]]]


def rejected_calls():
    """name -> (items, method, ws, ws_bytes, count): calls kfac_precondition rejects before it touches the device"""
    c = {}
    ok = item(DENSE, 300, 200)
    c['method_bad'] = ([ok], 0, FAKE_WS, SIZE_MAX, 1)
    c['count_negative'] = ([ok], _cabi.KFAC_EIGEN, FAKE_WS, SIZE_MAX, -1)
    c['items_null'] = (None, _cabi.KFAC_EIGEN, FAKE_WS, SIZE_MAX, 1)
    c['workspace_null'] = ([item(DENSE, 300, 200, qa=None)], _cabi.KFAC_EIGEN, None, SIZE_MAX, 1)
    c['workspace_small'] = ([ok], _cabi.KFAC_EIGEN, FAKE_WS, 4096, 1)
    for mname, m in METHODS.items():
        def add(name, items):
            c[f'{mname}_{name}'] = (items, m, FAKE_WS, SIZE_MAX, len(items))
        add('kind_bad', [item(7, 300, 200)])
        add('kind_negative', [ok, item(-1, 300, 200)])
        for kind, (g, a) in ((DENSE, (300, 200)), (EMB, (64, 3000)), (DIAG_G, (3000, 65)), (TIED, (64, 3000)),
                             (DIAG_A, (1100, 3001))):
            k = KIND_NAMES[kind]
            rows, cols = p_shape(kind, g, a)
            add(f'{k}_peers_many', [item(kind, g, a, n_peers=8, peer_P=C.cast(FAKE, C.POINTER(C.c_void_p)))])
            add(f'{k}_peers_null', [item(kind, g, a, n_peers=1)])
            add(f'{k}_peers_negative', [item(kind, g, a, n_peers=-1)])
            add(f'{k}_wgrad_null', [item(kind, g, a, wgrad=None)])
            add(f'{k}_P_null', [item(kind, g, a, P=None)])
            add(f'{k}_g0', [item(kind, 0, a)])
            add(f'{k}_a0', [item(kind, g, 0)])
            add(f'{k}_ldp_small', [item(kind, g, a, ldp=cols - 1)])
            add(f'{k}_ldp_small_not_ready', [item(kind, g, a, ldp=cols - 1, qa=None, qg=None, a_inv=None, g_inv=None)])
            for missing in not_ready(kind, mname):
                add(f'{k}_missing_{"_".join(missing)}', [item(kind, g, a, **{n: None for n in missing})])
            add(f'{k}_second_not_ready', [ok, item(kind, g, a, **{n: None for n in not_ready(kind, mname)[0]})])
            add(f'{k}_not_ready_then_bad', [item(kind, g, a, **{n: None for n in not_ready(kind, mname)[0]}),
                                            item(kind, g, a, wgrad=None)])
        add('dense_ldqa_small', [item(DENSE, 300, 200, ldqa=199)])
        add('dense_ldqg_small', [item(DENSE, 300, 200, ldqg=299)])
        add('dense_ldq_small_not_ready', [item(DENSE, 300, 200, ldqa=199, qa=None, a_inv=None)])
        add('dense_taps_negative', [item(DENSE, 300, 200, wgrad_taps=-1)])
        add('dense_taps_not_dividing', [item(DENSE, 300, 201, wgrad_taps=9)])
        add('dense_taps_not_dividing_bias', [item(DENSE, 300, 200, wgrad_taps=9, bgrad=FAKE)])
        add('dense_taps_ldq_small', [item(DENSE, 300, 200, wgrad_taps=-1, ldqg=1)])
        add('embedding_ldq_small', [item(EMB, 64, 3000, ldqg=63)])
        add('embedding_bias', [item(EMB, 64, 3000, bgrad=FAKE)])
        add('diag_g_ldq_small', [item(DIAG_G, 3000, 65, ldqa=64)])
        add('tied_ldq_small', [item(TIED, 64, 3000, ldqg=63)])
        add('tied_bias', [item(TIED, 64, 3000, bgrad=FAKE)])
        add('tied_damping_zero', [item(TIED, 64, 3000, tied_damping=0.0)])
        add('tied_damping_zero_not_ready', [item(TIED, 64, 3000, tied_damping=0.0, dh=None)])
        add('diag_a_ldq_small', [item(DIAG_A, 1100, 3001, ldqg=1099)])
        add('diag_a_ldp_g', [item(DIAG_A, 1100, 3001, ldp=1100)])
        add('mixed_last_bad', [item(DENSE, 300, 200), item(EMB, 64, 3000), item(DIAG_G, 3000, 65),
                               item(TIED, 64, 3000), item(DIAG_A, 1100, 3001), item(DIAG_A, 1100, 3001, P=None)])
    return c


def call(items, method, ws, ws_bytes, count):
    arr = array(items) if items is not None else None
    rc = lib().kfac_precondition(arr, count, method, 1e-3, ws, ws_bytes, None)
    return [rc, _cabi.last_error()]


def measure():
    ws = workspace_corpus()
    return {
        'workspace': {name: workspace_bytes(items) for name, items in ws.items()},
        'need': {name: {m: need(items, v) for m, v in METHODS.items()} for name, items in ws.items()},
        'rejected': {name: call(*args) for name, args in rejected_calls().items()},
    }


@pytest.fixture(scope='module')
def golden():
    with open(GOLDEN) as f:
        return json.load(f)


@pytest.mark.parametrize('name', sorted(workspace_corpus()))
def test_workspace_bytes(golden, name):
    """kfac_precondition_workspace_bytes covers either method: the eigen method's plans, which split the most"""
    items = workspace_corpus()[name]
    expect = golden['workspace'][name] - sum(unused_slab_bytes(it, 'eigen') for it in items)
    assert workspace_bytes(items) == expect


@pytest.mark.parametrize('method', sorted(METHODS))
@pytest.mark.parametrize('name', sorted(workspace_corpus()))
def test_call_needs_the_slabs_it_uses(golden, name, method):
    items = workspace_corpus()[name]
    expect = golden['need'][name][method] - sum(unused_slab_bytes(it, method) for it in items)
    assert need(items, METHODS[method]) == expect
    assert need(items, METHODS[method]) <= workspace_bytes(items)


@pytest.mark.parametrize('name', sorted(rejected_calls()))
def test_rejected_call(golden, name):
    """The same status and message, from the same check, before anything is launched"""
    assert call(*rejected_calls()[name]) == golden['rejected'][name]
    assert golden['rejected'][name][0] in (_cabi.KFAC_ERR_BAD_ARG, _cabi.KFAC_ERR_NOT_READY, _cabi.KFAC_ERR_WORKSPACE)


def main():
    out = sys.argv[1] if len(sys.argv) > 1 else GOLDEN
    res = measure()
    for name, (rc, _) in res['rejected'].items():
        assert rc in (_cabi.KFAC_ERR_BAD_ARG, _cabi.KFAC_ERR_NOT_READY, _cabi.KFAC_ERR_WORKSPACE), (name, rc)
    with open(out, 'w') as f:
        json.dump(res, f, indent=1, sort_keys=True)
        f.write('\n')
    print('wrote', out)


if __name__ == '__main__':
    main()
