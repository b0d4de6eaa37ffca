"""The lazy-exact Adam scheme of the fused hashed-table step (csrc/mf.cu slb_mf_bloom_train_step
under SLB_OPT_ADAM), restated in float64 for the CPU and GPU tests: oracle.bloom.step in dense mode
for the gradients, plus one oracle.adam.LazyAdamTable per table (user table, item table, user bias,
item bias), each with its own ``last``.

Step t: every table row the minibatch reads (the H rows of each user, positive and negative item,
the padding row included) and every bias of those ids is caught up through t - 1; the gradients are
taken from those tables; the rows and bias ids the oracle marks as touched take step t.

``mutate`` restates plausible kernel mistakes (tests/test_mf_bloom_adam_oracle_cpu.py shows that the
GPU tolerances catch each):

``prepass_no_negs``     the negatives' hashed item rows are not caught up before the forward
``bias_shares_last``    a bias reads its table's ``last`` (already advanced): it never catches up
``frozen_no_catch_up``  the frozen (padding) row is not caught up (it only moves at the flush)
``stash_post_update``   the item gradients are taken from the updated user rows
``bucket_merge``        distinct bias ids of one hash bucket merged (oracle.bloom's mutation)
"""

import numpy as np

from oracle import bloom as ob
from oracle.adam import LazyAdamTable

MUTATIONS = ('prepass_no_negs', 'bias_shares_last', 'frozen_no_catch_up', 'stash_post_update', 'bucket_merge')


def make_tables(P, lr, wd, betas=(0.9, 0.999), eps=1e-8):
    """[Wu, Wi, bu, bi] LazyAdamTables from the four (float) arrays."""
    return [LazyAdamTable(p, lr=lr, betas=betas, eps=eps, weight_decay=wd) for p in P]


def read_rows(case, Mu, Mi, users, items, negs):
    """(user table rows, item table rows, user ids, item ids) the step reads before its forward, for
    tables of Mu / Mi rows."""
    iids = np.concatenate([np.asarray(items).reshape(-1), np.asarray(negs).reshape(-1)])
    ru = ob.table_rows(users, case['Hu'], Mu, case['pad_u']).reshape(-1)
    ri = ob.table_rows(iids, case['Hi'], Mi, case['pad_i']).reshape(-1)
    return ru, ri, np.asarray(users).reshape(-1), iids


def lazy_step(tabs, case, users, items, negs, t, mutate=()):
    """One step t on ``tabs`` (modified in place); ``case`` carries loss, n_neg, Hu, Hi, pad_u and
    pad_i.  Returns oracle.bloom.step's dict for the step."""
    Wu, Wi, bu, bi = tabs
    users, items, negs = (np.asarray(x, dtype=np.int64).reshape(-1) for x in (users, items, negs))
    ru, ri, uid, iid = read_rows(case, Wu.w.shape[0], Wi.w.shape[0], users, items, negs)
    if 'prepass_no_negs' in mutate:
        ri = ob.table_rows(items, case['Hi'], Wi.w.shape[0], case['pad_i']).reshape(-1)
    for tab, rows, H, pad in ((Wu, ru, case['Hu'], case['pad_u']), (Wi, ri, case['Hi'], case['pad_i'])):
        fr = ob.frozen_row(H, pad)
        if 'frozen_no_catch_up' in mutate and fr >= 0:
            rows = rows[rows != fr]
        tab.catch_up(rows, t - 1)
    for tab, ids in ((bu, uid), (bi, iid)):
        if 'bias_shares_last' in mutate:
            tab.last[np.unique(ids)] = np.maximum(tab.last[np.unique(ids)], t - 1)
        else:
            tab.catch_up(ids, t - 1)
    P = [tab.w for tab in tabs]
    om = tuple(m for m in mutate if m in ob.MUTATIONS and m != 'stash_post_update')
    ref = ob.step([p.copy() for p in P], users, items, negs, case['loss'], case['Hu'], case['Hi'], case['pad_u'],
                  case['pad_i'], case['n_neg'], mutate=om)
    tWu, tWi, tbu, tbi = ref['touched']
    grads = [ref['dWu'], ref['dWi'], ref['dbu'], ref['dbi']]
    order = ((0, tWu), (2, tbu), (1, tWi), (3, tbi))
    for k, touched in order:
        if k == 1 and 'stash_post_update' in mutate:
            grads[1] = _item_grads(case, users, items, ref, Wu.w, Wi.w)
        rows = np.flatnonzero(touched)
        tabs[k].catch_up(rows, t - 1)          # a mutated prepass leaves rows behind: the apply catches up
        tabs[k].apply(rows, grads[k][rows], t)
    return ref


def _item_grads(case, users, items, ref, Wu, Wi):
    """The item-table gradient from the user table as it is now (the stash_post_update mistake)."""
    d = np.zeros(Wi.shape)
    sides = ((users, items, ref['gp']), (ref['kstar_user'], ref['kstar_item'], ref['gn']))
    for u, i, g in sides:
        ri = ob.table_rows(i, case['Hi'], Wi.shape[0], case['pad_i'])
        uv = Wu[ob.table_rows(u, case['Hu'], Wu.shape[0], case['pad_u'])].sum(axis=1)
        for k in range(ri.shape[1]):
            np.add.at(d, ri[:, k], g[:, None] * uv)
    fr = ob.frozen_row(case['Hi'], case['pad_i'])
    if fr >= 0:
        d[fr] = 0.0
    return d


def dense_adam(P, grads_fn, steps, lr, wd, betas=(0.9, 0.999), eps=1e-8):
    """Dense float64 Adam (torch.optim.Adam's formulas) over ``steps`` calls of grads_fn(P, t) ->
    four dense gradients; returns the tables."""
    P = [np.array(p, dtype=np.float64) for p in P]
    M = [np.zeros_like(p) for p in P]
    V = [np.zeros_like(p) for p in P]
    b1, b2 = betas
    for t in range(1, steps + 1):
        G = grads_fn(P, t)
        for p, m, v, g in zip(P, M, V, G):
            g = g + wd * p
            m += (g - m) * (1.0 - b1)
            v[:] = v * b2 + (1.0 - b2) * g * g
            p -= lr / (1.0 - b1 ** t) * (m / (np.sqrt(v) / np.sqrt(1.0 - b2 ** t) + eps))
    return P


def fixture_names(g):
    """state_dict names of (Wu, Wi, bu, bi) in a make_golden_bloom_adam.py fixture."""
    u = 'user_embeddings.embeddings.weight' if int(g['user_H']) else 'user_embeddings.weight'
    return [u, 'item_embeddings.embeddings.weight', 'user_biases.weight', 'item_biases.weight']


def fixture_case(g):
    """The hashing of a make_golden_bloom_adam.py fixture: loss, n_neg, Hu, Hi, pad_u, pad_i (the
    BloomEmbedding layers' padding id 0; a plain user table has none)."""
    loss, Hu = str(g['loss']), int(g['user_H'])
    return dict(loss=loss, n_neg=int(g['n_neg']) if loss == 'adaptive_hinge' else 1, Hu=Hu, Hi=int(g['item_H']),
                pad_u=0 if Hu else -1, pad_i=0)
