"""NCCL tests of the sharded (multi-GPU) paths on the product kernels.

Every case runs at world 1 -- the whole sharded code path (bucketing, all-to-alls
with itself, owner routing, score routing of the adaptive hinge) on one GPU, so a
single-GPU machine exercises it -- and at world 2 when two GPUs are visible.  One process group per world is spawned once per session and
runs all jobs; each test then checks its own job against the float64 oracle.
"""

import os
import sys

import numpy as np
import pytest
import torch

from conftest import ROOT, assert_close

sys.path.insert(0, os.path.join(ROOT, 'tests'))
pytestmark = pytest.mark.gpu

import sharded_common as sc            # noqa: E402

SHAPE = (7, 2000, 500, 32, 1024, 3)     # seed, U, I, D, B, steps
MF_JOBS = [('bpr', 'a2a'), ('pointwise', 'a2a'), ('bpr', 'dense')]

# tanh keeps the scores bounded: with relu at this scale the fp32 sigmoid saturates and a few
# row gradients underflow to exactly 0 where the float64 oracle keeps 1e-16, which Adagrad's
# first-touch normalisation turns into a full lr step (fp32 torch underflows the same way)
_CNN = dict(kernel_width=[3, 3], dilation=[1, 2], nonlinearity='tanh', residual=True)
SEQ_SHAPE = {'pool': (11, 300, 32, 24, 20, 3), 'cnn': (11, 300, 128, 24, 20, 3)}   # seed, I, D, B, S, steps
SEQ_JOBS = [('bpr', 'pool'), ('pointwise', 'cnn')]

FIT = dict(seed=33, U=3000, I=800, D=32, n=300000, B=16384, n_iter=2)
FIT_JOBS = [('bpr', 'a2a'), ('bpr', 'dense'), ('adaptive_hinge', 'a2a')]

ADA = dict(seed=19, U=1500, I=400, D=32, B=768, n=4)       # one adaptive-hinge step, gradients
BLOOM = (9, 3000, 40000, 1500, 32, 2048, 3, 4)            # seed, U, N ids, M hashed rows, D, B, steps, H


def _fit_problem():
    rs = np.random.RandomState(8)
    params, _ = sc.make_problem(6, FIT['U'], FIT['I'], FIT['D'], 8, 0)
    params = tuple(p * 0.3 for p in params)
    return params, rs.randint(0, FIT['U'], FIT['n']).astype(np.int32), rs.randint(0, FIT['I'], FIT['n']).astype(np.int32)


def _adaptive_grad_job(rank, world, dev):
    """One ShardedMF.step_adaptive on the product kernels with the gradients tapped where
    the step hands them to the optimizer (user side: scores_backward; item side: the rows
    each owner receives)."""
    from spotlight_b200.sharded import GpuBackend, ShardedMF, ShardPlan, ShardState

    class Tap(GpuBackend):
        def __init__(self, device):
            GpuBackend.__init__(self, device)
            self.rec = {}

        def scores_backward(self, st, cache_rows, g, u_idx, i_idx):
            out = GpuBackend.scores_backward(self, st, cache_rows, g, u_idx, i_idx)
            self.rec['dWu'] = out[0].cpu().numpy().copy()
            self.rec['dbu'] = out[2].reshape(-1).cpu().numpy().copy()
            return out

        def owner_update(self, st, local_ids, g_rows, g_bias):
            self.rec['ids'] = local_ids.cpu().numpy().copy()
            self.rec['g_rows'] = g_rows.cpu().numpy().copy()
            self.rec['g_bias'] = g_bias.cpu().numpy().copy()
            return GpuBackend.owner_update(self, st, local_ids, g_rows, g_bias)

    n = ADA['n']
    params, batches = sc.make_problem(ADA['seed'], ADA['U'], ADA['I'], ADA['D'], ADA['B'], 1, n_neg=n)
    users, items, negs = batches[0]
    plan = ShardPlan(ADA['U'], ADA['I'], world)
    st = ShardState(plan, rank, ADA['D'], dev, lr=0.05, init=[torch.from_numpy(p) for p in params])
    be = Tap(dev)
    model = ShardedMF(plan, st, rank, be)
    mine = np.nonzero(plan.user_owner(users) == rank)[0]
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(dev)      # noqa: E731
    loss = model.step_adaptive(t(users[mine]), t(items[mine]), t(negs.reshape(-1, n)[mine].reshape(-1)),
                               t(mine.astype(np.int64)), t(users), n)
    rec = dict(be.rec)
    rec.update(loss=float(loss), ulo=st.ulo, ilo=st.ilo)
    return rec


def _dense_stats_job(rank, world, dev):
    """fit() on the dense exchange (B = 16384 covers the 800 items twice over, so 'auto' picks it
    too), and one ShardedMF.step_dense on the same shards: the exchange stats of each."""
    from spotlight_b200.interactions import Interactions
    from spotlight_b200.sharded import GpuBackend, ShardedImplicitFactorizationModel, ShardedMF
    params, users, items = _fit_problem()
    model = ShardedImplicitFactorizationModel(FIT['U'], FIT['I'], rank, world, dev, loss='bpr',
                                              embedding_dim=FIT['D'], n_iter=FIT['n_iter'], batch_size=FIT['B'],
                                              random_state=np.random.RandomState(FIT['seed']), exchange='dense',
                                              init=[torch.from_numpy(p) for p in params])
    model.fit(Interactions(users, items, num_users=FIT['U'], num_items=FIT['I']))
    one = ShardedMF(model.plan, model.state, rank, GpuBackend(dev))
    empty = torch.zeros(0, dtype=torch.int64, device=dev)
    one.step_dense(empty, empty, empty, 'bpr', FIT['B'])
    return dict(model.mf.stats), dict(one.stats), model.plan.ichunk


def _jobs(rank, world, dev):
    from spotlight_b200.sharded import GpuBackend
    res = {}
    for loss, exchange in MF_JOBS:
        params, batches = sc.make_problem(*SHAPE)
        got, losses, stats = sc.sharded_run(rank, world, params, batches, loss, 0.05, dev,
                                            GpuBackend(dev), cache_capacity=min(2 * SHAPE[4], SHAPE[2]),
                                            exchange=exchange)
        res['mf', loss, exchange] = (got, losses)
    for loss, net in SEQ_JOBS:
        cnn = _CNN if net == 'cnn' else None
        params, batches = sc.make_seq_problem(*SEQ_SHAPE[net], layers=2 if cnn else 0)
        got, losses, stats = sc.seq_sharded_run(rank, world, params, batches, loss, 0.05, dev,
                                                GpuBackend(dev), cnn=cnn)
        res['seq', loss, net] = (got, losses)
    for loss, exchange in FIT_JOBS:
        params, users, items = _fit_problem()
        res['fit', loss, exchange] = sc.sharded_fit_run(rank, world, params, users, items, loss, dev,
                                                       GpuBackend(dev), FIT['seed'], FIT['B'],
                                                       FIT['n_iter'], exchange, n_neg=4)
    seed, U, N, M, D, B, steps, H = BLOOM
    params, batches = sc.make_bloom_problem(seed, U, N, M, D, B, steps)
    for loss in ('bpr', 'hinge'):
        res['bloom', loss] = sc.bloom_sharded_run(rank, world, params, batches, loss, 0.05, dev, GpuBackend(dev), H)
    res['ada', rank] = _adaptive_grad_job(rank, world, dev)
    res['dense_stats'] = _dense_stats_job(rank, world, dev)
    return res


_CACHE = {}


def _results(world):
    if torch.cuda.device_count() < world:
        pytest.skip('needs %d GPUs' % world)
    if world not in _CACHE:
        _CACHE[world] = sc.run_world(_jobs, world, backend='nccl', timeout=900)
    return _CACHE[world]


WORLDS = [1, 2]


@pytest.mark.parametrize('world', WORLDS)
@pytest.mark.parametrize('loss,exchange', MF_JOBS)
def test_sharded_gpu_matches_oracle(world, loss, exchange):
    got, losses = _results(world)[0]['mf', loss, exchange]
    params, batches = sc.make_problem(*SHAPE)
    ref, ref_losses = sc.oracle_run(params, batches, loss, 0.05)
    assert_close(np.array(losses), np.array(ref_losses), 1e-5, what='losses')
    for a, b, nm in zip(got, ref, ['Wu', 'Wi', 'bu', 'bi']):
        # Adagrad trajectory tolerance: first-touch normalisation amplifies 1e-7 gradient
        # differences on near-cancelling rows (see test_model_gpu / test_sharded_cpu)
        assert_close(a, b, 5e-3, what=nm)


@pytest.mark.parametrize('world', WORLDS)
@pytest.mark.parametrize('loss,net', SEQ_JOBS)
def test_sharded_sequence_gpu_matches_oracle(world, loss, net):
    got, losses = _results(world)[0]['seq', loss, net]
    cnn = _CNN if net == 'cnn' else None
    params, batches = sc.make_seq_problem(*SEQ_SHAPE[net], layers=2 if cnn else 0)
    ref, ref_losses = sc.seq_oracle_run(params, batches, loss, 0.05, cnn=cnn)
    assert_close(np.array(losses), np.array(ref_losses), 2e-5, what='losses')
    for k, (a, b) in enumerate(zip(got, ref)):
        assert_close(a, b, 5e-3, what='param%d' % k)      # Adagrad trajectory tolerance, as above


@pytest.mark.parametrize('world', WORLDS)
def test_sharded_adaptive_hinge_step_gradients(world):
    """One sharded adaptive-hinge step (reference pairing, implicit.py:266-275: flat negative
    f scored with users[f // n], consumed as element (f // B, f % B)) against the float64
    oracle: loss and all four gradients at the north star's 1e-5.  No trajectory, so none of
    the chaos that limits the fit() comparison below."""
    from oracle import mf as omf
    res = _results(world)
    n = ADA['n']
    params, batches = sc.make_problem(ADA['seed'], ADA['U'], ADA['I'], ADA['D'], ADA['B'], 1, n_neg=n)
    users, items, negs = batches[0]
    ref = omf.mf_step(*[p.astype(np.float64) for p in params], users, items, negs, 'adaptive_hinge', n,
                      np.float64)
    dWu = np.zeros_like(ref['dWu'])
    dbu = np.zeros(ADA['U'])
    dWi = np.zeros_like(ref['dWi'])
    dbi = np.zeros(ADA['I'])
    for r in range(world):
        rec = res[r]['ada', r]
        assert_close(rec['loss'], float(ref['loss']), 1e-5, what='loss')
        if 'dWu' in rec:
            dWu[rec['ulo']:rec['ulo'] + rec['dWu'].shape[0]] += rec['dWu']
            dbu[rec['ulo']:rec['ulo'] + rec['dbu'].shape[0]] += rec['dbu']
        np.add.at(dWi, rec['ilo'] + rec['ids'], rec['g_rows'].astype(np.float64))
        np.add.at(dbi, rec['ilo'] + rec['ids'], rec['g_bias'].astype(np.float64))
    assert_close(dWu, ref['dWu'], 1e-5, what='dWu')
    assert_close(dWi, ref['dWi'], 1e-5, what='dWi')
    assert_close(dbu, ref['dbu'].reshape(-1), 1e-5, atol=1e-9, what='dbu')
    assert_close(dbi, ref['dbi'].reshape(-1), 1e-5, atol=1e-9, what='dbi')
    assert np.abs(ref['dWi']).max() > 0 and np.abs(ref['dWu']).max() > 0


@pytest.mark.parametrize('world', WORLDS)
@pytest.mark.parametrize('loss', ['bpr', 'hinge'])
def test_sharded_bloom_gpu_matches_oracle(world, loss):
    """BASELINE config 4's partitioning on the product kernels (hashed item table range-sharded and
    exchanged whole, fused hashed step with in-register murmur3, sparse bias updates) against the
    single-process float64 oracle of BilinearNet + BloomEmbedding."""
    got, losses = _results(world)[0]['bloom', loss]
    seed, U, N, M, D, B, steps, H = BLOOM
    params, batches = sc.make_bloom_problem(seed, U, N, M, D, B, steps)
    ref, ref_losses = sc.bloom_oracle_run(params, batches, loss, 0.05, H)
    assert_close(np.array(losses), np.array(ref_losses), 1e-5, what='losses')
    for a, b, nm in zip(got, ref, ['Wu', 'Wi(hashed)', 'bu', 'bi']):
        if loss == 'hinge' and nm in ('bu', 'bi'):
            continue        # +-1/B gradients cancel exactly or leave a 1e-9 residue by summation order: see test_sharded_cpu
        assert_close(a, b.reshape(a.shape), 5e-3, what=nm)      # Adagrad trajectory tolerance


_SINGLE = {}


def _single_gpu_fit(loss):
    """The single-GPU product fit() from the same RandomState seed and weights."""
    if loss not in _SINGLE:
        import contextlib
        import io
        from spotlight_b200.factorization.implicit import ImplicitFactorizationModel
        from spotlight_b200.interactions import Interactions
        from spotlight_b200.optim import fused_adagrad
        params, users, items = _fit_problem()
        inter = Interactions(users, items, num_users=FIT['U'], num_items=FIT['I'])
        rs = np.random.RandomState(FIT['seed'])
        one = ImplicitFactorizationModel(loss=loss, embedding_dim=FIT['D'], n_iter=FIT['n_iter'],
                                         batch_size=FIT['B'], use_cuda=True, random_state=rs,
                                         num_negative_samples=4,
                                         optimizer_func=fused_adagrad(lr=0.05))
        one._initialize(inter)
        net = one._net
        with torch.no_grad():
            for prm, val in zip((net.user_embeddings.weight, net.item_embeddings.weight,
                                 net.user_biases.weight, net.item_biases.weight), params):
                prm.copy_(torch.from_numpy(val).to(prm.device).reshape(prm.shape))
        buf = io.StringIO()
        with contextlib.redirect_stdout(buf):
            one.fit(inter, verbose=True)
        losses = [float(line.split('loss')[1]) for line in buf.getvalue().splitlines()
                  if line.startswith('Epoch')]
        ref = [p.detach().cpu().numpy() for p in (net.user_embeddings.weight, net.item_embeddings.weight,
                                                  net.user_biases.weight, net.item_biases.weight)]
        _SINGLE[loss] = (ref, losses, rs.get_state())
    return _SINGLE[loss]


@pytest.mark.parametrize('world', WORLDS)
@pytest.mark.parametrize('loss,exchange', FIT_JOBS)
def test_sharded_fit_equals_single_gpu_fit(world, loss, exchange):
    """N-GPU fit() vs the single-GPU product fit() from the same RandomState seed and
    weights: same permutation (device shuffle, n >= 2^17), same negatives, same minibatches
    -> same final tables, same final generator state."""
    got, losses, state = _results(world)[0]['fit', loss, exchange]
    ref, single_losses, want = _single_gpu_fit(loss)
    # adaptive hinge across ranks: the owners sum their peers' gradient rows in rank order, a
    # different (equally valid) fp32 order than one GPU's -- exactly the kind of 1e-7 perturbation
    # that this trajectory amplifies (see below; the oracle's own epoch losses move 1.7e-5 under it)
    loss_tol = 1e-4 if (loss == 'adaptive_hinge' and world > 1) else 2e-5
    assert_close(np.array(losses), np.array(single_losses), loss_tol, what='epoch losses')
    for a, b, nm in zip(got, ref, ['Wu', 'Wi', 'bu', 'bi']):
        if loss == 'adaptive_hinge':
            # This trajectory is chaotic at the row level: in the float64 oracle a 1e-7 relative
            # perturbation of the initial item table moves every user row by more than 1.6e-3
            # (max 0.05 on a 0.32 scale) within these two epochs, while the epoch losses move by
            # < 2e-5 (profiles/adaptive_sensitivity.py).  The two GPU paths score with different
            # kernels (fused tile forward vs mf_scores), i.e. differ by such a perturbation.  The
            # step itself is held to 1e-5 in test_sharded_adaptive_hinge_step_gradients; the exact
            # trajectory semantics are pinned on the CPU against the oracle
            # (tests/test_sharded_cpu.py, worlds 2 and 3).  Here: finite, and correlated.
            floor = {'Wu': 0.8, 'Wi': 0.3}.get(nm)
            assert np.isfinite(a).all()
            if floor is not None:
                assert np.corrcoef(a.reshape(-1), b.reshape(-1))[0, 1] > floor, nm
        else:
            assert_close(a, b.reshape(a.shape), 5e-3, what=nm)   # Adagrad trajectory tolerance, as above
    assert np.array_equal(state[1], want[1]) and state[2] == want[2]
    assert len(losses) == FIT['n_iter'] and all(0.0 < v < 1.5 for v in losses)


@pytest.mark.parametrize('world', WORLDS)
def test_sharded_dense_epoch_counts_the_exchange(world):
    """The dense-exchange epoch counts, on every rank and for every step, what ShardedMF.step_dense
    counts: the whole padded item table (world * ichunk rows) requested, and the table, its bias and
    their gradients moved as float32."""
    steps = FIT['n_iter'] * -(-FIT['n'] // FIT['B'])
    for r in range(world):
        fit_stats, step_stats, chunk = _results(world)[r]['dense_stats']
        assert step_stats == {'rows_requested': world * chunk,
                              'bytes_a2a': 2 * (world * chunk * FIT['D'] + world * chunk) * 4}
        assert fit_stats == {k: steps * v for k, v in step_stats.items()}
