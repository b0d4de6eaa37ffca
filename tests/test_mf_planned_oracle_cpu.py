"""The cases and tolerances of tests/test_mf_planned_oracle_gpu.py, checked without a GPU.

* Every matrix case carries the member-list length classes, hot rows and score scales it
  promises (oracle/mf_cases.py).
* oracle.mf.fit reproduces the live reference's fit trajectory (tests/golden/fit_bpr_sgd.npz,
  D = 8, B = 64: the planned route), which pins the float64 oracle to the reference.
* Each plausible planned-step mistake, restated as a mutated oracle call on a suite case, moves
  the update, the state change, the handed-out gradient or the loss by more than the GPU
  suite's 1e-5 tolerance.
"""

import numpy as np
import pytest

from conftest import assert_close, load_golden
from oracle import mf as omf
from oracle import mf_cases as mc

DIMS = (8, 16, 32, 64, 128)


@pytest.mark.parametrize('D', DIMS)
@pytest.mark.parametrize('size', ['small', 'large'])
def test_suite_cases_have_their_properties(D, size):
    for loss in mc.LOSSES:
        case = (mc.small_case if size == 'small' else mc.large_case)(D, loss)
        ref = omf.fused_step(mc.tables64(case), case['users'], case['items'], case['negs'], loss, 'sgd', 0.0)
        assert mc.check_properties(case, ref) == [], (D, size, loss)
        lens = mc.member_lengths(case)
        cap, G = mc.seg_sort_cap(D), mc.long_groups(D)
        assert cap == {8: 32, 16: 64}.get(D, 128)
        for side in ('user', 'item'):
            for name, lo, hi in mc.length_classes(D)[side]:
                assert ((lens[side] >= lo) & (lens[side] <= hi)).any(), (side, name)
            assert ((lens[side] > cap + 1) & (lens[side] % G != 0)).any()


def test_determinism_case_spreads_hot_users_over_scan_tiles():
    case = mc.make_case(64, 30000, 'bpr', seed=41, extra_hot_users=40, min_users=300_000)
    lens = np.bincount(case['users'], minlength=case['U'])
    hot = np.flatnonzero(lens > case['cap'])
    assert len(hot) >= 41 and len(np.unique(hot // 4096)) >= 30


def test_fit_reproduces_reference_trajectory():
    g = load_golden('fit_bpr_sgd')
    names = ['user_embeddings.weight', 'item_embeddings.weight', 'user_biases.weight', 'item_biases.weight']
    P = [g['init.' + k].astype(np.float64) for k in names]
    rs = np.random.RandomState(int(g['seed']))
    rs.randint(-10 ** 8, 10 ** 8)                 # the model constructor's draw (implicit.py:114)
    losses = omf.fit(P, g['users'], g['items'], int(g['num_items']), 'bpr', int(g['batch']), int(g['n_iter']),
                     rs, 'sgd', 0.5)
    assert_close(np.array(losses), g['epoch_losses'], 1e-5, what='epoch losses')
    for p, k in zip(P, names):
        assert_close(p, g['final.' + k], 1e-5, atol=1e-8, what=k)
    st = rs.get_state()
    assert (st[1] == g['rs_key']).all() and st[2] == int(g['rs_pos'])


def outcome(case, opt, wd_on, mutate=(), norm=None):
    """What the GPU suite compares: loss, the update and state change of every table, the
    handed-out item gradient."""
    lr, wd, S0 = mc.hparams(case, opt, wd_on)
    P0 = mc.tables64(case)
    P = [p.copy() for p in P0]
    S = [s.astype(np.float64) for s in S0] if S0 else None
    out = omf.fused_step(P, case['users'], case['items'], case['negs'], case['loss'], opt, lr, wd, 1e-10, S,
                         norm=norm, mutate=mutate, cap=case['cap'])
    res = dict(loss=np.array(out['loss']), dWi=out['dWi'], dbi=out['dbi'])
    for k, nm in enumerate(('Wu', 'Wi', 'bu', 'bi')):
        res[nm] = P[k] - P0[k]
        if S:
            res['s' + nm] = S[k] - S0[k]
    return res


def differs(ref, mut, keys=None):
    """True when at least one compared quantity misses the GPU suite's 1e-5."""
    for k in keys or ref:
        try:
            assert_close(mut[k], ref[k], 1e-5, what=k)
        except AssertionError:
            return True
    return False


def caught(case, opt, wd_on, mutation, keys=None, norm=None):
    return differs(outcome(case, opt, wd_on, norm=norm), outcome(case, opt, wd_on, (mutation,), norm=norm), keys)


@pytest.mark.parametrize('D', [8, 64])
def test_catches_item_side_reading_post_update_user_rows(D):
    assert caught(mc.small_case(D, 'bpr'), 'sgd', False, 'stash_post_update', ('Wi', 'bi'))


@pytest.mark.parametrize('D', [16, 128])
def test_catches_negative_term_credited_to_positive_row(D):
    assert caught(mc.small_case(D, 'hinge'), 'adagrad', False, 'neg_to_pos_row', ('Wi', 'bi'))


def test_catches_user_bias_gradient_without_gn():
    assert caught(mc.small_case(32, 'pointwise'), 'sgd', False, 'user_bias_no_gn', ('bu',))


@pytest.mark.parametrize('D', [8, 128])
def test_catches_hinge_strict_inequality_at_the_tie(D):
    """Only the z = 0 interaction differs: its user row and both its item rows."""
    case = mc.small_case(D, 'hinge')
    assert caught(case, 'sgd', False, 'hinge_strict', ('Wu',))
    assert caught(case, 'sgd', False, 'hinge_strict', ('bi',))


@pytest.mark.parametrize('opt', ['sgd', 'adagrad'])
def test_catches_decay_on_rows_without_a_term(opt):
    """The inactive hinge user and its item rows have no non-zero term: they stay."""
    assert caught(mc.small_case(32, 'hinge'), opt, True, 'decay_all_rows', ('Wu', 'Wi', 'bu', 'bi'))


@pytest.mark.parametrize('mutation,keys', [('no_decay_user_rows', ('Wu',)), ('no_decay_biases', ('bu',)),
                                           ('no_decay_biases', ('bi',))])
@pytest.mark.parametrize('opt', ['sgd', 'adagrad'])
def test_catches_decay_skipped(mutation, keys, opt):
    assert caught(mc.small_case(64, 'bpr'), opt, True, mutation, keys)


@pytest.mark.parametrize('D', [8, 128])
def test_catches_adagrad_dividing_before_adding(D):
    assert caught(mc.small_case(D, 'pointwise'), 'adagrad', True, 'adagrad_div_before_add', ('Wu', 'Wi', 'bu', 'bi'))


@pytest.mark.parametrize('D', [8, 32, 128])
def test_catches_item_lists_summing_only_four_terms(D):
    assert caught(mc.small_case(D, 'bpr'), 'sgd', False, 'item_first4', ('Wi', 'bi'))


@pytest.mark.parametrize('D', [8, 64])
@pytest.mark.parametrize('side', ['user', 'item'])
def test_catches_last_member_of_hot_list_dropped(D, side):
    keys = ('Wu', 'bu') if side == 'user' else ('Wi', 'bi')
    assert caught(mc.small_case(D, 'pointwise'), 'adagrad', False, 'hot_drop_last', keys)


def test_catches_gradient_out_normalised_by_local_batch():
    case = mc.small_case(64, 'bpr')
    assert caught(case, 'sgd', False, 'local_norm', ('dWi',), norm=3 * case['B'])
    assert caught(case, 'adagrad', False, 'local_norm', ('loss',), norm=3 * case['B'])


def test_unmutated_outcome_is_self_consistent():
    """Sanity of the comparison itself: the same call twice does not differ, and the update of
    an SGD step equals -lr * (g + wd * w) on touched rows."""
    case = mc.small_case(16, 'hinge')
    a, b = outcome(case, 'sgd', True), outcome(case, 'sgd', True)
    assert not differs(a, b)
    lr, wd, _ = mc.hparams(case, 'sgd', True)
    P = mc.tables64(case)
    out = omf.fused_step([p.copy() for p in P], case['users'], case['items'], case['negs'], 'hinge', 'sgd', lr, wd)
    tu = out['touched_u']
    assert_close(a['Wu'][tu], -lr * (out['dWu'][tu] + wd * P[0][tu]), 1e-12)
    assert (a['Wu'][~tu] == 0).all() and (~tu).sum() > 0
