"""The hashed-table oracle (oracle/bloom.py) and the cases of tests/test_mf_bloom_oracle_gpu.py,
checked without a GPU.

* oracle.bloom reproduces the live reference: the Bloom-item-layer step fixtures and a two-epoch
  fit() with a Bloom item layer and Adagrad (tests/golden/fit_bloom_adagrad.npz).
* With plain tables it is oracle.mf.fused_step (the planned step's rule), and with a plain user
  table it is oracle.mf.mf_bloom_step.
* Every matrix case carries the ids, term counts and score scales it promises.
* Each plausible kernel mistake, restated as a mutated oracle call, moves the update, the state
  change, a gradient or the loss by more than the GPU suite's 1e-5 tolerance.
"""

import numpy as np
import pytest

from conftest import assert_close, load_golden
from oracle import bloom as ob
from oracle import bloom_cases as bc
from oracle import mf as omf

TABLES = ('Wu', 'Wi', 'bu', 'bi')


@pytest.mark.parametrize('name,loss', [('mf_hinge_bloom', 'hinge'), ('mf_adaptive_bloom', 'adaptive_hinge')])
def test_reproduces_reference_step_fixtures(name, loss):
    g = load_golden(name)
    H = int(g['bloom_H'])
    n = int(g['n_neg']) if loss == 'adaptive_hinge' else 1
    names = ['user_embeddings.weight', 'item_embeddings.embeddings.weight', 'user_biases.weight',
             'item_biases.weight']
    P = [g['sd.' + k].astype(np.float64) for k in names]
    out = ob.step(P, g['users'], g['items'], g['negs'], loss, 0, H, -1, 0, n)
    assert_close(out['pos'], g['pos'], 1e-5, what='pos')
    assert_close(out['neg'].reshape(g['neg'].shape), g['neg'], 1e-5, what='neg')
    assert_close(out['loss'], g['loss'], 1e-5, what='loss')
    for k, nm in zip(names, ('dWu', 'dWi', 'dbu', 'dbi')):
        assert_close(out[nm], g['grad.' + k], 1e-5, atol=1e-8, what=nm)


def test_fit_reproduces_reference_trajectory():
    """Two epochs of the reference's fit() with a Bloom item layer and torch.optim.Adagrad
    (wd = 0: the row-wise fused Adagrad is the dense one)."""
    g = load_golden('fit_bloom_adagrad')
    names = ['user_embeddings.weight', 'item_embeddings.embeddings.weight', 'user_biases.weight',
             'item_biases.weight']
    P = [g['init.' + k].astype(np.float64) for k in names]
    S = [np.zeros(p.shape) for p in P]
    rs = np.random.RandomState()
    rs.set_state(('MT19937', g['rs0_key'], int(g['rs0_pos'])))
    losses = ob.fit(P, g['users'], g['items'], int(g['num_items']), 'bpr', int(g['batch']), int(g['n_iter']), rs,
                    'adagrad', float(g['lr']), Hu=0, Hi=int(g['bloom_H']), pad_i=0, states=S)
    assert_close(np.array(losses), g['epoch_losses'], 1e-5, what='epoch losses')
    for p, k in zip(P, names):
        assert_close(p, g['final.' + k], 1e-5, atol=1e-7, what=k)
    st = rs.get_state()
    assert (st[1] == g['rs_key']).all() and st[2] == int(g['rs_pos'])
    # predict(3): every item's score for user 3 from the final tables
    rows = ob.table_rows(np.arange(int(g['num_items'])), int(g['bloom_H']), P[1].shape[0], 0)
    u = int(g['predict_user'])
    pred = P[1][rows].sum(1) @ P[0][u] + P[2][u, 0] + P[3][:, 0]
    assert_close(pred, g['predict'], 1e-5, what='predict')


@pytest.mark.parametrize('loss', ['pointwise', 'bpr', 'hinge'])
@pytest.mark.parametrize('opt,wd', [('sgd', 0.1), ('adagrad', 0.1)])
def test_plain_tables_are_the_planned_rule(loss, opt, wd):
    case = bc.make_case(32, loss, 0, 0, -1, seed=5)
    P1, P2 = bc.tables64(case), bc.tables64(case)
    S1 = [np.full(p.shape, 1e-3) for p in P1] if opt == 'adagrad' else None
    S2 = [s.copy() for s in S1] if S1 else None
    a = ob.step(P1, case['users'], case['items'], case['negs'], loss, opt=opt, lr=0.05, weight_decay=wd, states=S1)
    b = omf.fused_step(P2, case['users'], case['items'], case['negs'], loss, opt, 0.05, wd, 1e-10, S2)
    assert_close(a['loss'], b['loss'], 1e-12)
    for x, y in zip(P1 + (S1 or []), P2 + (S2 or [])):
        assert_close(x, y, 1e-12)


@pytest.mark.parametrize('loss', ['pointwise', 'bpr', 'hinge'])
def test_plain_users_are_mf_bloom_step(loss):
    case = bc.make_case(16, loss, 0, 3, 0, seed=6)
    P = bc.tables64(case)
    a = ob.step(P, case['users'], case['items'], case['negs'], loss, 0, 3, -1, 0)
    b = omf.mf_bloom_step(*P, case['users'], case['items'], case['negs'], loss, 3, 0)
    for k in ('loss', 'pos', 'neg', 'dWu', 'dWi', 'dbu', 'dbi'):
        assert_close(a[k], b[k], 1e-12, atol=1e-15, what=k)       # bpr's gp + gn: summed in another order


@pytest.mark.parametrize('entry', bc.matrix(), ids=lambda e: '%d-%s%d-%d,%d-pad%d' % e[:6])
def test_matrix_cases_have_their_properties(entry):
    case = bc.case_for(*entry)
    assert bc.check_properties(case, bc.scores(case)) == []


def test_large_batch_case():
    case = bc.make_case(128, 'bpr', 0, 4, 0, seed=77, B=9000)
    assert case['B'] > 8448 and bc.check_properties(case, bc.scores(case)) == []


def outcome(case, opt, wd_on, mutate=()):
    """What the GPU suite compares: the loss and the update / state change of every table (fused),
    and the dense gradients."""
    lr, wd, S0 = bc.hparams(case, opt, wd_on)
    P0 = bc.tables64(case)
    P = [p.copy() for p in P0]
    S = [s.astype(np.float64) for s in S0] if S0 else None
    args = (case['users'], case['items'], case['negs'], case['loss'], case['Hu'], case['Hi'], case['pad_u'],
            case['pad_i'], case['n_neg'])
    out = ob.step(P, *args, opt=opt, lr=lr, weight_decay=wd, states=S, mutate=mutate)
    dense = ob.step(bc.tables64(case), *args, mutate=mutate)
    res = dict(loss=np.array(out['loss']), pos=dense['pos'], neg=dense['neg'])
    for k, nm in enumerate(TABLES):
        res[nm] = P[k] - P0[k]
        res['d' + nm] = dense['d' + nm]
        if S:
            res['s' + nm] = S[k] - S0[k]
    return res


def differs(ref, mut):
    for k in ref:
        try:
            assert_close(mut[k], ref[k], 1e-5, what=k)
        except AssertionError:
            return True
    return False


# (mutation, case entry, opt, wd_on): a case and optimizer on which the mistake shows
CATCH = [
    ('pad_hashed', (32, 'bpr', 1, 0, 4, 0, 11), 'sgd', False),
    ('freeze_row0', (20, 'pointwise', 1, 2, 3, 3, 12), 'sgd', False),
    ('train_frozen', (20, 'pointwise', 1, 2, 3, 3, 12), 'adagrad', False),
    ('item_first_hash', (8, 'bpr', 1, 0, 4, -1, 13), 'sgd', False),
    ('item_mean', (64, 'hinge', 1, 0, 24, 0, 14), 'sgd', False),
    ('dup_row_once', (12, 'pointwise', 1, 2, 3, -1, 15), 'sgd', False),
    ('adaptive_user_b', (32, 'adaptive_hinge', 5, 0, 4, 3, 16), 'sgd', False),
    ('last_tie', (48, 'adaptive_hinge', 2, 0, 1, 0, 17), 'sgd', False),
    ('stash_post_update', (32, 'bpr', 1, 3, 0, 0, 18), 'sgd', False),
    ('user_bias_no_gn', (100, 'adaptive_hinge', 2, 2, 3, -1, 19), 'sgd', False),
    ('user_bias_zero_pair', (64, 'bpr', 1, 0, 4, 0, 20), 'adagrad', True),
    ('user_bias_zero_pair', (24, 'hinge', 1, 2, 3, 3, 21), 'sgd', True),
    ('decay_all_rows', (32, 'hinge', 1, 0, 1, -1, 22), 'sgd', True),
    ('adagrad_div_before_add', (128, 'pointwise', 1, 0, 0, -1, 23), 'adagrad', True),
    ('bucket_merge', (16, 'pointwise', 1, 0, 1, 0, 24), 'sgd', False),
    ('drop_last_pair', (256, 'bpr', 1, 0, 4, 3, 25), 'adagrad', False),
]


def test_every_mutation_has_a_catch():
    assert {m for m, *_ in CATCH} == set(ob.MUTATIONS)


@pytest.mark.parametrize('mutation,entry,opt,wd_on', CATCH, ids=['%s-%d' % (c[0], k) for k, c in enumerate(CATCH)])
def test_catches_mutation(mutation, entry, opt, wd_on):
    case = bc.case_for(*entry)
    assert bc.check_properties(case, bc.scores(case)) == []
    ref = outcome(case, opt, wd_on)
    assert not differs(ref, outcome(case, opt, wd_on))
    assert differs(ref, outcome(case, opt, wd_on, (mutation,)))
