"""World-size-2 (and 3) gloo tests of the multi-GPU routing logic on CPU: the
sharded step (bucketing -> all-to-all -> gather -> all-to-all -> local step ->
all-to-all -> owner update -> all-reduce) with a NumPy backend must reproduce
the single-process oracle step on the concatenated batch.

Hinge is not used for the trajectory comparison: its gradients are +-1/B, so a
bias row hit by as many positives as negatives has an *exactly* cancelling
gradient in one summation order and a 1e-18 residue in another, which
Adagrad's first-touch normalisation turns into a full +-lr step (the same
sign-level sensitivity the reference has between any two summation orders)."""

import os
import sys

import numpy as np
import pytest
import torch

from conftest import ROOT, assert_close

sys.path.insert(0, os.path.join(ROOT, 'tests'))

import sharded_common as sc            # noqa: E402


def _step_job(rank, world, dev, loss, exchange):
    params, batches = sc.make_problem(5, 101, 57, 8, 96, 3)
    return sc.sharded_run(rank, world, params, batches, loss, 0.05, dev, sc.NumpyBackend(), exchange=exchange)


@pytest.mark.parametrize('world,loss,exchange', [(2, 'bpr', 'a2a'), (3, 'bpr', 'a2a'),
                                                 (2, 'pointwise', 'a2a'), (2, 'bpr', 'dense'),
                                                 (3, 'pointwise', 'dense')])
def test_sharded_step_matches_single_process(world, loss, exchange):
    got, losses, stats = sc.run_world(_step_job, world, (loss, exchange))[0]
    params, batches = sc.make_problem(5, 101, 57, 8, 96, 3)
    ref, ref_losses = sc.oracle_run(params, batches, loss, 0.05)
    assert_close(np.array(losses), np.array(ref_losses), 1e-5, what='losses')
    for a, b, nm in zip(got, ref, ['Wu', 'Wi', 'bu', 'bi']):
        assert_close(a, b, 2e-5, what=nm)
    # each distinct row crosses the wire once per rank per step, never per use
    if exchange == 'a2a':
        assert stats['rows_requested'] <= 3 * 57


_CNN = dict(kernel_width=[3, 3], dilation=[1, 2], nonlinearity='tanh', residual=True)


def _seq_job(rank, world, dev, loss, net):
    cnn = _CNN if net == 'cnn' else None
    params, batches = sc.make_seq_problem(9, 41, 8, 10, 7, 3, layers=2 if cnn else 0)
    return sc.seq_sharded_run(rank, world, params, batches, loss, 0.05, dev, sc.NumpyBackend(), cnn=cnn)


@pytest.mark.parametrize('world,loss,net', [(2, 'bpr', 'pool'), (3, 'pointwise', 'pool'),
                                            (2, 'bpr', 'cnn')])
def test_sharded_sequence_step_matches_single_process(world, loss, net):
    """Sequence models (SURVEY §8e, config 5): sequences are data-parallel, item rows
    range-sharded and fetched once per step, conv weights replicated + all-reduced,
    loss normalised by the global unmasked count."""
    got, losses, stats = sc.run_world(_seq_job, world, (loss, net))[0]
    cnn = _CNN if net == 'cnn' else None
    params, batches = sc.make_seq_problem(9, 41, 8, 10, 7, 3, layers=2 if cnn else 0)
    ref, ref_losses = sc.seq_oracle_run(params, batches, loss, 0.05, cnn=cnn)
    assert_close(np.array(losses), np.array(ref_losses), 1e-5, what='losses')
    assert len(got) == len(ref)
    for k, (a, b) in enumerate(zip(got, ref)):
        assert_close(a, b, 3e-5, what='param%d' % k)
    assert stats['rows_requested'] <= 3 * 41
    assert not got[0][0].any() and not got[1][0].any()          # padding row stays zero


FIT = dict(seed=21, U=61, I=37, D=8, n=500, B=64, n_iter=2)


def _fit_problem():
    rs = np.random.RandomState(4)
    params, _ = sc.make_problem(5, FIT['U'], FIT['I'], FIT['D'], 8, 0)
    users = rs.randint(0, 40, FIT['n']).astype(np.int32)          # world 3: rank 2 owns users >= 42, always empty
    items = rs.randint(0, FIT['I'], FIT['n']).astype(np.int32)
    return params, users, items


def _fit_job(rank, world, dev, loss, exchange):
    params, users, items = _fit_problem()
    return sc.sharded_fit_run(rank, world, params, users, items, loss, dev, sc.NumpyBackend(),
                              FIT['seed'], FIT['B'], FIT['n_iter'], exchange, n_neg=3)


@pytest.mark.parametrize('world,loss,exchange', [(2, 'bpr', 'a2a'), (3, 'pointwise', 'dense'),
                                                 (2, 'adaptive_hinge', 'a2a'), (3, 'adaptive_hinge', 'a2a')])
def test_sharded_fit_is_the_single_process_fit(world, loss, exchange):
    """fit() on N ranks forms the reference's minibatches from the reference's RandomState
    stream (global shuffle, one randint per minibatch), so its trajectory is the
    single-process one; with 500 interactions in minibatches of 64 over 3 ranks some ranks
    get empty shares, which must not stall the collectives."""
    got, losses, state = sc.run_world(_fit_job, world, (loss, exchange))[0]
    params, users, items = _fit_problem()
    n_neg = 3 if loss == 'adaptive_hinge' else 1
    epochs, rs = sc.reference_epochs(FIT['seed'], users, items, FIT['I'], FIT['B'], FIT['n_iter'], n_neg)
    flat = [b for e in epochs for b in e]
    ref, ref_losses = sc.oracle_run(params, flat, loss, 0.05, n_neg=n_neg)
    per_epoch = np.array(ref_losses).reshape(FIT['n_iter'], -1).mean(axis=1)
    assert_close(np.array(losses), per_epoch, 1e-5, what='epoch losses')
    for a, b, nm in zip(got, ref, ['Wu', 'Wi', 'bu', 'bi']):
        assert_close(a, b, 5e-5, what=nm)
    want = rs.get_state()
    assert np.array_equal(state[1], want[1]) and state[2] == want[2]      # stream position too


SEEDED = dict(seed=23, U=90, I=37, D=8, n=500, B=64, n_iter=2)


def _seeded_problem(users_in):
    p = SEEDED
    params = sc.make_margin_params(6, p['U'], p['I'], p['D'])
    rs = np.random.RandomState(12)
    users = rs.randint(0, users_in, p['n']).astype(np.int32)
    items = rs.randint(0, p['I'], p['n']).astype(np.int32)
    S0 = sc.seeded_accumulators(7, params, sc.accumulator_scales(p['B']))
    return params, users, items, S0


def _seeded_fit_job(rank, world, dev, loss, users_in):
    p = SEEDED
    params, users, items, S0 = _seeded_problem(users_in)
    return sc.sharded_fit_run(rank, world, params, users, items, loss, dev, sc.NumpyBackend(), p['seed'], p['B'],
                              p['n_iter'], 'dense', S0=S0)


@pytest.mark.parametrize('loss,users_in', [('bpr', SEEDED['U']), ('hinge', SEEDED['U']), ('pointwise', 40)])
def test_seeded_accumulator_replay_is_the_sharded_fit(loss, users_in):
    """The float64 replay the GPU tests hold the dense-exchange fit() to -- oracle_run from seeded
    accumulators over reference_epochs' minibatches -- is the sharded fit() of the NumPy backend
    at world 2 with I odd: the changes of all four tables and their accumulators, relative to the
    largest change, the epoch losses and the final RandomState agree; the padded row of the last
    item shard keeps its zeros and its accumulator bit for bit.  users_in = 40 puts every user in
    rank 0's range, so rank 1 serves item rows with no members of its own."""
    p = SEEDED
    res = sc.run_world(_seeded_fit_job, 2, (loss, users_in))
    got, losses, state, (acc, _) = res[0]
    params, users, items, S0 = _seeded_problem(users_in)
    epochs, rs = sc.reference_epochs(p['seed'], users, items, p['I'], p['B'], p['n_iter'])
    margins = []
    ref, ref_losses, ref_acc = sc.oracle_run(params, [b for e in epochs for b in e], loss, 0.05, S0=S0,
                                             each=lambda r: margins.append(sc.hinge_margin(r)))
    if loss == 'hinge':
        assert min(margins) > 1e-4
    per_epoch = np.array(ref_losses).reshape(p['n_iter'], -1).mean(axis=1)
    assert_close(np.array(losses), per_epoch, 1e-5, what='epoch losses')
    for nm, e in sc.change_errors(got + acc, ref + ref_acc, list(params) + S0, loss, 0.05).items():
        assert e <= 1e-5, (nm, e)
    want = rs.get_state()
    assert np.array_equal(state[1], want[1]) and state[2] == want[2]
    W, S, b, sb = res[1][3][1]                               # rank 1: 19 rows for 18 items
    assert W.shape[0] == 1 and not W.any() and not b.any()
    assert np.all(S == 1.0) and np.all(sb == 1.0)


def test_shard_plan_ranges():
    from spotlight_b200.sharded import ShardPlan
    plan = ShardPlan(10, 7, 4)
    assert [plan.user_range(r) for r in range(4)] == [(0, 3), (3, 6), (6, 9), (9, 10)]
    assert [plan.item_range(r) for r in range(4)] == [(0, 2), (2, 4), (4, 6), (6, 7)]
    assert plan.user_owner(torch.tensor([0, 2, 3, 9])).tolist() == [0, 0, 1, 3]


BLOOM = (9, 120, 700, 64, 8, 128, 3, 3)         # seed, U, N ids, M hashed rows, D, B, steps, H


def _bloom_job(rank, world, dev, loss):
    seed, U, N, M, D, B, steps, H = BLOOM
    params, batches = sc.make_bloom_problem(seed, U, N, M, D, B, steps)
    return sc.bloom_sharded_run(rank, world, params, batches, loss, 0.05, dev, sc.NumpyBackend(), H)


@pytest.mark.parametrize('world,loss', [(2, 'bpr'), (3, 'pointwise'), (4, 'bpr')])
def test_sharded_bloom_step_matches_single_process(world, loss):
    """BASELINE config 4's partitioning (hashed item rows range-sharded, users owner-routed,
    id-space item bias replicated through all-gathered sparse updates) against the
    single-process float64 oracle of BilinearNet + BloomEmbedding."""
    got, losses = sc.run_world(_bloom_job, world, (loss,))[0]
    seed, U, N, M, D, B, steps, H = BLOOM
    params, batches = sc.make_bloom_problem(seed, U, N, M, D, B, steps)
    ref, ref_losses = sc.bloom_oracle_run(params, batches, loss, 0.05, H)
    assert_close(np.array(losses), np.array(ref_losses), 1e-5, what='losses')
    for a, b, nm in zip(got, ref, ['Wu', 'Wi(hashed)', 'bu', 'bi']):
        assert_close(a, b.reshape(a.shape), 2e-5, what=nm)

