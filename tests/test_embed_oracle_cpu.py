"""The generic route's oracle (oracle/embed.py) and the cases of tests/test_embed_oracle_gpu.py,
checked without a GPU.

* The restatements agree with plain NumPy on small cases (np.add.at scatter, torch-free
  bilinear scores), the ordered float32 forms with the float64 ones at the GPU suite's 1e-6.
* Every matrix case carries the widths, segment lengths, ids and score ranges it promises.
* Each plausible kernel mistake, restated as a mutated oracle call, moves a compared quantity
  past the GPU suite's tolerance on some case (``order_desc``: the ordered float32 bits).
"""

import numpy as np
import pytest

from conftest import assert_close
from oracle import embed as oe
from oracle import embed_cases as ec
from oracle import mf as omf
from oracle.murmur import bloom_rows

MATRIX = ec.matrix()
IDS = [ec.entry_id(e) for e in MATRIX]
LOOKUP_TOL, OTHER_TOL = 1e-6, 1e-5
_CASES = {}


def case_of(entry):
    if entry not in _CASES:
        _CASES[entry] = ec.case_for(entry)
    return _CASES[entry]


def test_lookup_restates_numpy():
    rs = np.random.RandomState(0)
    W = ec.values(rs, (11, 6))
    dout = ec.values(rs, (50, 6))
    for H, pad in ((0, -1), (0, 3), (3, 0), (3, 4)):
        ids_ = rs.randint(0, 11 if H == 0 else 40, 50)
        rows = ids_[:, None] if H == 0 else bloom_rows(ids_, H, 11, pad)
        assert_close(oe.lookup(W, ids_, H, pad), W.astype(np.float64)[rows].sum(1), 1e-15)
        want = np.zeros((11, 6))
        for k in range(rows.shape[1]):
            np.add.at(want, rows[:, k], dout.astype(np.float64))
        if pad >= 0:
            want[pad] = 0
        assert_close(oe.lookup_backward(dout, ids_, H, 11, pad), want, 1e-15)
        # the ordered float32 sum of a row, added by hand in term order
        got = oe.lookup_backward(dout, ids_, H, 11, pad, ordered=True)
        r = rows.reshape(-1)
        for row in range(11):
            acc = np.float32(0)
            for t in np.flatnonzero(r == row):
                acc = np.float32(acc + dout[t // rows.shape[1], 0])
            assert got[row, 0] == (0 if row == pad else acc)


def test_scores_restate_bilinear():
    case = ec.scores_case(12, 301, 'batch', 1)
    s = oe.scores(case['Wu'], case['Wi'], case['bu'], case['bi'], case['users'], case['items'])
    want = omf.bilinear_scores(case['Wu'], case['Wi'], case['bu'], case['bi'], case['users'], case['items'],
                               np.float64)
    assert_close(s, want, 1e-15)
    # the backward is the transpose of the forward: <g, d s / d Wu> by finite differences
    dWu, dWi, dbu, dbi = oe.scores_backward(case['g'], case['Wu'], case['Wi'], case['users'], case['items'])
    Wu = case['Wu'].astype(np.float64)
    E = np.zeros_like(Wu)
    E[17, 3] = 1e-3
    fd = (oe.scores(Wu + E, case['Wi'], case['bu'], case['bi'], case['users'], case['items']) - s) @ case['g']
    assert abs(fd / 1e-3 - dWu[17, 3]) < 1e-9 * max(1.0, abs(dWu[17, 3]))


def test_broadcast_is_a_repeated_user():
    case = ec.scores_case(8, 101, 'bcast', 2)
    rep = np.full(101, case['users'][0])
    a = oe.scores_backward(case['g'], case['Wu'], case['Wi'], case['users'], case['items'])
    b = oe.scores_backward(case['g'], case['Wu'], case['Wi'], rep, case['items'])
    for x, y in zip(a, b):
        assert_close(x, y, 1e-15)


@pytest.mark.parametrize('entry', MATRIX, ids=IDS)
def test_matrix_cases_have_their_properties(entry):
    case = case_of(entry)
    assert ec.check_properties(case) == []
    if case['kind'] == 'lookup':
        # the ordered float32 restatement is within the GPU suite's float64 tolerance
        ref, o, bound = ec.oracle(case), ec.ordered(case), ec.sum_bounds(case)
        for k in ('out', 'dW'):
            assert ec.within(o[k], ref[k], bound[k], LOOKUP_TOL) is None, k


def test_every_width_instantiation_is_reached():
    """(LPR, VEC4) of emb_fwd_kernel / emb_bwd_kernel over the lookup cases: all twelve."""
    seen = {(oe.pow2_lanes(e[1]), oe.vec4(e[1])) for e in MATRIX if e[0] in ('segments', 'hashed')}
    assert seen == {(l, v) for l in (1, 2, 4, 8, 16, 32) for v in (False, True)}
    assert any(e[1] > 32 * (4 if oe.vec4(e[1]) else 1) for e in MATRIX if e[0] == 'segments')


def differs(case, mutation):
    """Whether the mutated float64 oracle leaves what the GPU suite compares with a tolerance:
    lookups at 1e-6 plus the float32 summation bound, hashed rows exactly, the rest at 1e-5."""
    ref, mut = ec.oracle(case), ec.oracle(case, (mutation,))
    if case['kind'] == 'lookup':
        bound = ec.sum_bounds(case)
        return (not np.array_equal(ref['rows'], mut['rows'])
                or any(ec.within(mut[k], ref[k], bound[k], LOOKUP_TOL) for k in ('out', 'dW')))
    for k in ref:
        try:
            assert_close(mut[k], ref[k], OTHER_TOL, what=k)
        except AssertionError:
            return True
    return False


# (mutation, matrix entry): a case on which the mistake shows
CATCH = [
    ('pad_hashed', ('hashed', 5, 24, 0, 203)),
    ('freeze_row0', ('segments', 3, 5, 102)),
    ('train_frozen', ('segments', 2, 0, 101)),
    ('dup_row_once', ('tiny', 3, 2, 0, 1, 301)),
    ('fan_mod', ('hashed', 2, 2, 5, 201)),
    ('fan_mod', ('hashed', 3, 4, -1, 202)),
    ('tail_zero', ('segments', 33, 5, 108)),
    ('tail_zero', ('segments', 100, 0, 116)),
    ('long_drop_last', ('segments', 1, -1, 100)),
    ('long_drop_last', ('segments', 512, 5, 120)),
    ('bcast_user_once', ('scores', 12, 1001, 'bcast', 613)),
    ('last_tie', ('pairwise', 'adaptive_hinge', 5, 257, 'random', 743)),
    ('mask_mean_over_n', ('pairwise', 'bpr', 1, 255, 'single', 711)),
]
ORDER_CATCH = [('segments', 1, -1, 100), ('segments', 64, -1, 115)]


def test_every_mutation_has_a_catch():
    assert {m for m, _ in CATCH} | {'order_desc'} == set(oe.MUTATIONS)
    for _, e in CATCH:
        assert e in MATRIX, e
    for e in ORDER_CATCH:
        assert e in MATRIX, e


@pytest.mark.parametrize('mutation,entry', CATCH, ids=['%s-%d' % (c[0], k) for k, c in enumerate(CATCH)])
def test_catches_mutation(mutation, entry):
    assert differs(case_of(entry), mutation)


@pytest.mark.parametrize('entry', ORDER_CATCH, ids=[ec.entry_id(e) for e in ORDER_CATCH])
def test_descending_order_changes_bits(entry):
    """order_desc leaves the float64 result within tolerance but flips float32 bits."""
    case = case_of(entry)
    assert not differs(case, 'order_desc')
    a, b = ec.ordered(case)['dW'], ec.ordered(case, ('order_desc',))['dW']
    assert (a.view(np.int32) != b.view(np.int32)).any()
