"""The event-to-event matcher on the device (esvo_em_match, esvo_b200/csrc/em.cu) against the oracle on every case of
tests/em_cases.py, bit for bit: the accepted set, the thread-major order, every seed field including the cost, and the number
of ZNCC evaluations.  Both back-project with the reference's literal cam2World (4x4 cofactor inverse), sum the patches
row-major and sequentially and contract no a*b+c, so nothing is left to a tolerance; the integer-rig cases put every warp
exactly on a pixel boundary, where any other rounding of cam2World picks other patches and other border decisions."""
import numpy as np
import pytest

import em_cases as E
from esvo_b200 import capi, configs
from test_em_pins import EXACT_COST_BOUND, exact_cost_errors

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def contexts(oracle_lib, product_lib):
    """(oracle_for, product_for): one context per rig and library; the oracle one also holds the product's own rig tables."""
    cache = {}

    def get(lib, rig):
        if (lib.path, rig) not in cache:
            l, r = configs.rig_calibs(rig)
            be = capi.Backend(lib, l, r, E.params(rig, lib))
            if lib is oracle_lib:
                for cam, c in ((0, l), (1, r)):
                    be.set_rectify_tables(cam, *capi.compute_rectify_tables(product_lib, c))
            cache[(lib.path, rig)] = be
        return cache[(lib.path, rig)]
    return (lambda rig: get(oracle_lib, rig)), (lambda rig: get(product_lib, rig))


@pytest.fixture(scope="module")
def runs(contexts):
    """case id -> (inputs, kw, oracle seeds, oracle evaluations, product seeds, product evaluations)."""
    oracle_for, product_for = contexts
    cache = {}

    def get(cid):
        if cid not in cache:
            c = E.CASES[cid]
            inp = E.case_inputs(c, oracle_for)
            kw = E.case_kw(c)
            so, eo = E.run(E.load_case(oracle_for(inp["rig"]), inp), inp, kw)
            sg, eg = E.run(E.load_case(product_for(inp["rig"]), inp), inp, kw)
            cache[cid] = (inp, kw, so, eo, sg, eg)
        return cache[cid]
    return get


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint8)


@pytest.mark.parametrize("cid", list(E.CASES))
def test_event_matcher_case_bit_identical(runs, cid):
    inp, kw, so, eo, sg, eg = runs(cid)
    print(cid, "matches", so.size, sg.size, "evaluations", eo, eg)
    assert eg == eo, "ZNCC evaluations"
    assert sg.size == so.size, "accepted set"
    assert np.array_equal(sg["t_ns"], so["t_ns"]), "event order"
    for f in capi.SEED_DTYPE.names:
        assert np.array_equal(_bits(sg[f]), _bits(so[f])), f


def test_device_cost_is_within_bound_of_exact(runs):
    """The mpmath evaluation of tests/test_em_pins.py on the device's seeds."""
    errs = exact_cost_errors(lambda cid: (lambda r: (r[0], r[1], r[4], r[5], None))(runs(cid)))
    print("pairs", errs.size, "max |f64 - exact|", errs.max())
    assert errs.size >= 500 and errs.max() <= EXACT_COST_BOUND


@pytest.mark.parametrize("cid", ["q-borders-15x7", "nt7-total513"])
def test_capacity_contract(contexts, runs, cid):
    """Too small a capacity returns ESVO_ERR_CAPACITY with the count (on both libraries); capacity 0 with no buffer is the
    count query."""
    inp, kw, so, eo, sg, eg = runs(cid)
    for be_for in contexts:
        be = E.load_case(be_for(inp["rig"]), inp)
        assert E.em_match_raw(be, inp, kw, so.size - 1) == (-4, so.size, eo)
        assert E.em_match_raw(be, inp, kw, 0, with_buffer=False) == (-4, so.size, eo)
        assert E.em_match_raw(be, inp, kw, so.size) == (0, so.size, eo)
