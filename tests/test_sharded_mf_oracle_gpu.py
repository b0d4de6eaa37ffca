"""ShardedMF steps and the dense-exchange fit() epoch on the product kernels against the float64
oracle, from seeded Adagrad accumulators.

From zero accumulators Adagrad's first step is about lr * sign(g) whatever g's magnitude, which
hides most errors in g and forces a loose tolerance on the trajectory.  Here every accumulator
starts positive (sharded_common.seeded_accumulators, at the gradients' own scale; hot rows at
theirs, sharded_common.scale_hot_row), so each update
is -lr g / sqrt(S0 + g^2), smooth in g, and the changes of the parameters and accumulators (value
after minus value at start) are held to the oracle's changes relative to the largest of them --
tight enough to catch a dropped or misrouted gradient term.

The row spaces span several of segindex.cuh's 4096-row scan tiles; the step cases have a hot item
with more positions than any lane group's in-register sort and a hot user; the fit() cases run the
dense-exchange epoch (_epoch_dense_gpu: member gather, planned step in phases on two plan slots,
reduce-scatter, owner-shard Adagrad) at a mid shape and at the benchmark's shape.  NCCL through
sharded_common.run_world: world 1 always (the collectives are identities but every kernel of the
route runs), world 2 when two GPUs are visible; one process group per world runs all jobs."""

import os
import sys

import numpy as np
import pytest
import torch

from conftest import ROOT, assert_close

sys.path.insert(0, os.path.join(ROOT, 'tests'))
pytestmark = pytest.mark.gpu

import sharded_common as sc            # noqa: E402

LR = 0.05
RTOL = 1e-5                            # changes, relative to the oracle's largest change
NAMES = sc.TABLE_NAMES

STEP = dict(seed=17, U=20000, I=3 * 4096 + 17, B=8192, steps=3, hot_item=4096, hot_user=8192)
STEP_JOBS = [(exchange, loss, D) for exchange in ('a2a', 'dense') for loss in ('bpr', 'pointwise', 'hinge')
             for D in (32, 64)]

MID = dict(seed=41, U=50000, I=3 * 4096 + 17, D=64, B=65536, n=5 * 65536 - 1000)
BENCH = dict(seed=43, U=1000000, I=100000, D=64, B=524288, n=3 * 524288 - 1000)
FIT_JOBS = [('mid', 'bpr', 1), ('mid', 'pointwise', 1), ('mid', 'hinge', 1), ('mid', 'bpr', 2),
            ('bench', 'bpr', 1)]
SHAPES = {'mid': MID, 'bench': BENCH, 'rank0': MID}


# ------------------------------------------------------------------ problems


def _step_problem(D):
    """Tables, three minibatches (a tenth of the positives on one item just past a scan-tile edge,
    far more than seg_sort_cap's 128; a twentieth of the members on one user) and accumulators."""
    p = STEP
    params = sc.make_margin_params(p['seed'], p['U'], p['I'], D)
    rs = np.random.RandomState(p['seed'] + 1)
    batches = []
    for _ in range(p['steps']):
        users = rs.randint(0, p['U'], p['B'])
        users[rs.rand(p['B']) < 0.05] = p['hot_user']
        items = rs.randint(0, p['I'], p['B'])
        items[rs.rand(p['B']) < 0.1] = p['hot_item']
        batches.append((users.astype(np.int64), items.astype(np.int64),
                        rs.randint(0, p['I'], p['B']).astype(np.int64)))
    S0 = sc.seeded_accumulators(p['seed'] + 2, params, sc.accumulator_scales(p['B']))
    sc.scale_hot_row(S0, 0, p['hot_user'], 0.05 * p['B'])
    sc.scale_hot_row(S0, 1, p['hot_item'], 0.1 * p['B'])
    return params, batches, S0


def _fit_problem(shape):
    """Tables, interactions (a twentieth of them on item 4096) and accumulators; 'rank0' puts every
    user in rank 0's range of a world-2 plan."""
    p = SHAPES[shape]
    params = sc.make_margin_params(p['seed'], p['U'], p['I'], p['D'])
    rs = np.random.RandomState(p['seed'] + 1)
    users = rs.randint(0, p['U'] // 2 if shape == 'rank0' else p['U'], p['n']).astype(np.int32)
    items = rs.randint(0, p['I'], p['n']).astype(np.int32)
    items[rs.rand(p['n']) < 0.05] = 4096
    S0 = sc.seeded_accumulators(p['seed'] + 2, params, sc.accumulator_scales(p['B']))
    sc.scale_hot_row(S0, 1, 4096, 0.05 * p['B'])
    return params, users, items, S0


# ------------------------------------------------------------------ the jobs (every rank)


def _step_job(rank, world, dev, exchange, loss, D):
    """Three ShardedMF.step calls from seeded accumulators: the tables and accumulators after the
    first and after the last, the losses and this rank's padded item rows."""
    from spotlight_b200.sharded import GpuBackend, ShardedMF, ShardPlan, ShardState
    p = STEP
    params, batches, S0 = _step_problem(D)
    plan = ShardPlan(p['U'], p['I'], world)
    st = ShardState(plan, rank, D, dev, lr=LR, init=[torch.from_numpy(x) for x in params])
    sc.seed_accumulators(st, S0)
    model = ShardedMF(plan, st, rank, GpuBackend(dev))
    snaps, losses = [], []
    for k, (users, items, negs) in enumerate(batches):
        mine = plan.user_owner(users) == rank
        t = lambda x: torch.from_numpy(x[mine]).to(dev)        # noqa: E731
        losses.append(float(model.step(t(users), t(items), t(negs), loss, len(users), exchange)))
        if k in (0, len(batches) - 1):
            snaps.append(sc.gather_tables(st, plan, p['U'], p['I']) +
                         sc.gather_accumulators(st, plan, p['U'], p['I']))
    return snaps, losses, sc.padded_rows(st)


def _fit_job(rank, world, dev, shape, loss, n_iter):
    from spotlight_b200.sharded import GpuBackend
    p = SHAPES[shape]
    params, users, items, S0 = _fit_problem(shape)
    tables, losses, state, (acc, pad) = sc.sharded_fit_run(rank, world, params, users, items, loss, dev,
                                                           GpuBackend(dev), p['seed'], p['B'], n_iter, 'dense',
                                                           S0=S0)
    return tables + acc, losses, state, pad


def _jobs(rank, world, dev):
    res = {}
    for job in STEP_JOBS:
        res['step', job] = _step_job(rank, world, dev, *job)
    for job in FIT_JOBS + ([('rank0', 'bpr', 1)] if world == 2 else []):
        res['fit', job] = _fit_job(rank, world, dev, *job)
    return res


_CACHE = {}


def _results(world):
    if torch.cuda.device_count() < world:
        pytest.skip('needs %d GPUs' % world)
    if world not in _CACHE:
        _CACHE[world] = sc.run_world(_jobs, world, backend='nccl', timeout=1800)
    return _CACHE[world]


def _check_changes(got, ref, start, what, loss, rtol=RTOL):
    errs = sc.change_errors(got, ref, start, loss, LR)
    print('%s: max change error %s' % (what, ', '.join('%s %.2e' % kv for kv in errs.items())))
    k = int(np.argmax([errs[nm] for nm in NAMES[:4]]))
    idx, w0, dg, dr = sc.worst_change(got[k], ref[k], start[k])
    print('    worst %s%s: start %.6e, change %.6e, oracle change %.6e, S0 %.6e, oracle S %.6e'
          % (NAMES[k], idx, w0, dg, dr, start[k + 4].reshape(np.shape(ref[k]))[idx], ref[k + 4][idx]))
    for nm, e in errs.items():
        k = NAMES.index(nm)
        assert e <= rtol, '%s %s: change error %.3e > %.0e at (index, start, change, oracle change) %s' % (
            what, nm, e, rtol, sc.worst_change(got[k], ref[k], start[k]))


WORLDS = [1, 2]


@pytest.mark.parametrize('world', WORLDS)
@pytest.mark.parametrize('exchange,loss,D', STEP_JOBS)
def test_sharded_mf_steps_match_oracle_from_seeded_accumulators(world, exchange, loss, D):
    """One and three ShardedMF.step calls (per-row and dense exchange) against oracle_run from the
    same accumulators: losses at 1e-5, the changes of all four tables and their accumulators at
    1e-5 of the largest change."""
    from spotlight_b200.sharded import ShardPlan
    res = _results(world)
    snaps, losses, _ = res[0]['step', (exchange, loss, D)]
    params, batches, S0 = _step_problem(D)
    start = list(params) + S0
    margins = []
    ref, ref_losses, ref_S = sc.oracle_run(params, batches, loss, LR, S0=S0,
                                           each=lambda r: margins.append(sc.hinge_margin(r)))
    if loss == 'hinge':
        # an fp32-versus-float64 flip at the kink would be a false failure: the seed leaves none near it
        assert min(margins) > 1e-4, min(margins)
    assert_close(np.array(losses), np.array(ref_losses), 1e-5, what='losses')
    one, one_losses, one_S = sc.oracle_run(params, batches[:1], loss, LR, S0=S0)
    _check_changes(snaps[0], one + one_S, start, '%s/%s/D%d step 1' % (exchange, loss, D), loss)
    _check_changes(snaps[1], ref + ref_S, start, '%s/%s/D%d step 3' % (exchange, loss, D), loss)
    plan = ShardPlan(STEP['U'], STEP['I'], world)
    W, S, b, sb = res[world - 1]['step', (exchange, loss, D)][2]
    assert W.shape[0] == world * plan.ichunk - STEP['I']
    assert not W.any() and not b.any() and np.all(S == 1.0) and np.all(sb == 1.0)


_REPLAY = {}


def _replay(shape, loss, n_iter):
    """The float64 replay of the reference's minibatches and negatives from the seeded accumulators:
    (tables + accumulators, epoch losses, final RandomState, smallest hinge margin, start)."""
    key = shape, loss, n_iter
    if key not in _REPLAY:
        p = SHAPES[shape]
        params, users, items, S0 = _fit_problem(shape)
        epochs, rs = sc.reference_epochs(p['seed'], users, items, p['I'], p['B'], n_iter)
        del users, items
        nb = len(epochs[0])
        margins = []
        ref, ref_losses, ref_S = sc.oracle_run(params, [b for e in epochs for b in e], loss, LR, S0=S0,
                                               each=lambda r: margins.append(sc.hinge_margin(r)))
        per_epoch = np.array(ref_losses).reshape(n_iter, nb).mean(axis=1)
        _REPLAY.clear()                                     # the benchmark shape's replay is large: keep one
        _REPLAY[key] = (ref + ref_S, per_epoch, rs.get_state(), min(margins), list(params) + S0, nb)
    return _REPLAY[key]


def _check_fit(world, job):
    shape, loss, n_iter = job
    from spotlight_b200.sharded import ShardPlan
    p = SHAPES[shape]
    res = _results(world)
    got, losses, state, _ = res[0]['fit', job]
    ref, per_epoch, want, margin, start, nb = _replay(shape, loss, n_iter)
    if loss == 'hinge':
        assert margin > 1e-4, margin
    assert len(losses) == n_iter
    assert_close(np.array(losses), per_epoch, 1e-5, what='epoch losses')
    _check_changes(got, ref, start, '%s/%s/%d epochs (%d steps each)' % (shape, loss, n_iter, nb), loss)
    assert np.array_equal(state[1], want[1]) and state[2] == want[2]
    plan = ShardPlan(p['U'], p['I'], world)
    W, S, b, sb = res[world - 1]['fit', job][3]
    assert W.shape[0] == world * plan.ichunk - p['I']
    assert not W.any() and not b.any() and np.all(S == 1.0) and np.all(sb == 1.0)


@pytest.mark.parametrize('world', WORLDS)
@pytest.mark.parametrize('shape,loss,n_iter', FIT_JOBS)
def test_sharded_dense_fit_matches_oracle_from_seeded_accumulators(world, shape, loss, n_iter):
    """fit() on the dense exchange against the float64 replay of the reference's minibatches and
    negatives (reference_epochs) from the same accumulators.  'mid': U = 50000, I = 3 * 4096 + 17,
    D = 64, B = 65536, five steps with a short last one, so both plan slots are reused (and with
    n_iter = 2 the epoch buffers too); 'bench': the benchmark's shape, U = 1M, I = 100K, D = 64,
    B = 524288, three steps.  Epoch losses at 1e-5, the changes of the four tables and their
    accumulators at 1e-5 of the largest change, the final RandomState equal, and at world 2 (I odd)
    the padded row of the last item shard untouched bit for bit."""
    _check_fit(world, (shape, loss, n_iter))


def test_sharded_dense_fit_with_an_idle_rank_matches_oracle():
    """World 2, every user in rank 0's range: rank 1 has no members in any minibatch and only serves
    its item shard, and the tables and epoch losses still match the replay."""
    _check_fit(2, ('rank0', 'bpr', 1))
