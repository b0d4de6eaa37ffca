"""GPU tests of sharded sequence training with row-wise lazy-exact Adam on the product kernels:
the owner-side Adam entries (slb_shard_rows_adam_catch_up, slb_shard_rows_adam) against
oracle.adam.LazyAdamTable, ShardedSeq steps against the float64 dense-Adam oracle (NCCL, world 1
always, world 2 when two GPUs are visible), and ShardedImplicitSequenceModel.fit() with fused_adam
at world 1 against the single-GPU ImplicitSequenceModel with fused_adam on the same data and seed."""

import contextlib
import io
import os
import sys

import numpy as np
import pytest
import torch

from conftest import ROOT, assert_close

sys.path.insert(0, os.path.join(ROOT, 'tests'))
pytestmark = pytest.mark.gpu

import sharded_common as sc                  # noqa: E402
import test_sharded_seq_adam_cpu as tac      # noqa: E402
import test_sharded_seq_gpu as tsg           # noqa: E402
from oracle.adam import LazyAdamTable        # noqa: E402
from test_sharded_seq_cpu import gather_state, owner_case  # noqa: E402

DEV = torch.device('cuda', 0)
T = 6                # the step the kernel tests take; rows start current for earlier steps


# ------------------------------------------------------------------ owner-side Adam kernels

def _kernel_case(kind, D, seed=7, rows=300):
    """Request lists of four peers (one empty) concatenated in rank order, so rows repeat across
    requesters, with Adam state from earlier steps and rows current for different steps.
    'hot': one row at 300 positions (past any lane group's in-register sort); 'tiles': the same over
    a row space of several 4096-row scan tiles, the hot row just past a tile edge; 'zero': rows
    whose every received gradient row and bias is zero."""
    peers, hot_row = (90, 0, 140, 50), 7
    if kind == 'tiles':
        rows, peers, hot_row = 3 * 4096 + 17, (900, 0, 1400, 500), 4096
    ids, g_rows, g_bias, W, _, b, _ = owner_case(seed, rows, D, peers=peers, padding=3)
    rs = np.random.RandomState(seed + 1)
    if kind in ('hot', 'tiles'):
        ids = np.concatenate([ids, np.full(300, hot_row, dtype=np.int64)])
        g_rows = np.concatenate([g_rows, rs.randn(300, D).astype(np.float32)])
        g_bias = np.concatenate([g_bias, rs.randn(300).astype(np.float32)])
    if kind == 'zero':
        quiet = np.isin(ids, np.unique(ids[ids >= 0])[::5])
        g_rows[quiet] = 0
        g_bias[quiet] = 0
    m = (rs.randn(rows, D) * 0.1).astype(np.float32)
    v = (np.abs(rs.randn(rows, D)) * 0.01).astype(np.float32)
    bm = (rs.randn(rows) * 0.1).astype(np.float32)
    bv = (np.abs(rs.randn(rows)) * 0.01).astype(np.float32)
    last = rs.randint(0, T, rows).astype(np.int32)
    m[last == 0] = v[last == 0] = 0              # never stepped: no moments yet
    bm[last == 0] = bv[last == 0] = 0
    return ids, g_rows, g_bias, [W, m, v, b, bm, bv, last]


def _oracle(case, wd):
    ids, g_rows, g_bias, (W, m, v, b, bm, bv, last) = case
    tabs = []
    for w, mm, vv in ((W, m, v), (b, bm, bv)):
        tab = LazyAdamTable(w, lr=1e-2, weight_decay=wd)
        tab.m, tab.v = mm.astype(np.float64), vv.astype(np.float64)
        tab.last = last.astype(np.int64)
        tabs.append(tab)
    keep = ids >= 0
    rows = np.unique(ids[keep])
    slot = np.searchsorted(rows, ids[keep])
    dW, db = np.zeros((len(rows), W.shape[1])), np.zeros(len(rows))
    np.add.at(dW, slot, g_rows[keep].astype(np.float64))
    np.add.at(db, slot, g_bias[keep].astype(np.float64))
    for tab, g in zip(tabs, (dW, db)):
        tab.catch_up(rows, T - 1)
        tab.apply(rows, g, T)
    return [tabs[0].w, tabs[0].m, tabs[0].v, tabs[1].w, tabs[1].m, tabs[1].v, tabs[0].last]


def _sched():
    from spotlight_b200.optim import FusedAdam
    return FusedAdam([torch.zeros(1)], lr=1e-2).schedule(T, DEV)


def _run_kernels(case, wd, catch_up=True):
    from spotlight_b200 import _lib, ops
    lib = _lib.load()
    ids, g_rows, g_bias, tensors = case
    t = [torch.from_numpy(x.copy()).to(DEV) for x in tensors]
    d_ids, d_g, d_gb = (torch.from_numpy(x).to(DEV) for x in (ids, g_rows, g_bias))
    rows, D = t[0].shape
    sched = _sched()
    tail = [ops._ptr(x) for x in t] + [rows, D, ops._ptr(sched), T, 0.9, 0.999, 0.1, 1.0 - 0.999, 1e-8, wd]
    R = len(ids)
    if catch_up:
        _lib.check(lib.slb_shard_rows_adam_catch_up(ops._ptr(d_ids), R, *tail, ops._stream()), 'catch_up')
    need = lib.slb_shard_rows_workspace_bytes(R, rows)
    ws = torch.zeros(need, dtype=torch.uint8, device=DEV)
    _lib.check(lib.slb_shard_rows_adam(ops._ptr(d_ids), ops._ptr(d_g), ops._ptr(d_gb), R, *tail, ops._ptr(ws), need,
                                       ops._stream()), 'shard_rows_adam')
    torch.cuda.synchronize()
    return [x.cpu().numpy() for x in t]


NAMES = ('W', 'exp_avg', 'exp_avg_sq', 'bias', 'bias exp_avg', 'bias exp_avg_sq')


@pytest.mark.parametrize('wd', [0.0, 1e-2])
@pytest.mark.parametrize('kind', ['peers', 'hot', 'zero', 'tiles'])
@pytest.mark.parametrize('D', [3, 16, 128, 256])
def test_owner_adam_kernels_match_lazy_adam(D, kind, wd):
    """Catch-up then step T on every distinct requested row (rank-order sums of duplicates across
    requesters, -1 padding slots, a hot row, all-zero gradient rows; D = 3 takes the scalar rows):
    table, moments and bias at fp32 rounding of LazyAdamTable's float64, `last` exact; untouched rows
    bit for bit; two runs bit-identical; the step alone (no catch-up ahead of it) gives the same to
    fp32 rounding."""
    case = _kernel_case(kind, D)
    want = _oracle(case, wd)
    got = _run_kernels(case, wd)
    for g, w, nm in zip(got[:6], want[:6], NAMES):
        # 1e-5: the hot row's 300-term fp32 sum, squared into exp_avg_sq, is the largest value there
        assert_close(g, w, 1e-5, atol=1e-7, what=nm)
    assert np.array_equal(got[6], want[6].astype(np.int32))
    ids = case[0]
    untouched = np.setdiff1d(np.arange(got[0].shape[0]), ids)
    assert len(untouched) > 0
    for g, x in zip(got, case[3]):
        assert np.array_equal(g[untouched], x[untouched])
    for g, a in zip(got, _run_kernels(case, wd)):
        assert np.array_equal(g, a)
    alone = _run_kernels(case, wd, catch_up=False)
    for g, a, nm in zip(got[:6], alone[:6], NAMES):
        assert_close(a, g, 1e-6, atol=1e-8, what=nm + ' (step alone)')
    assert np.array_equal(got[6], alone[6])


def test_owner_adam_kernels_empty_and_rejections():
    """R == 0 changes nothing and needs no storage; null pointers, bad sizes and steps, rows for an
    empty shard and a short workspace are rejected before any launch."""
    from spotlight_b200 import _lib, ops
    lib = _lib.load()
    ids, g_rows, g_bias, tensors = _kernel_case('peers', 8)
    t = [torch.from_numpy(x.copy()).to(DEV) for x in tensors]
    d = [torch.from_numpy(x).to(DEV) for x in (ids, g_rows, g_bias)]
    sched = _sched()
    stream = ops._stream()
    R, rows = len(ids), t[0].shape[0]
    scal = [0.9, 0.999, 0.1, 1.0 - 0.999, 1e-8, 0.0]
    nulls = [None] * 7
    assert lib.slb_shard_rows_adam_catch_up(None, 0, *nulls, 0, 8, None, T, *scal, stream) == 0
    assert lib.slb_shard_rows_adam(None, None, None, 0, *nulls, 0, 8, None, T, *scal, None, 0, stream) == 0
    need = lib.slb_shard_rows_workspace_bytes(R, rows)
    ws = torch.zeros(need, dtype=torch.uint8, device=DEV)
    P = ops._ptr

    def args(**bad):
        a = dict(ids=P(d[0]), g=P(d[1]), gb=P(d[2]), R=R, W=P(t[0]), m=P(t[1]), v=P(t[2]), b=P(t[3]), bm=P(t[4]),
                 bv=P(t[5]), last=P(t[6]), rows=rows, dim=8, sched=P(sched), step=T, ws=P(ws), wsb=need)
        a.update(bad)
        tabs = [a[k] for k in ('W', 'm', 'v', 'b', 'bm', 'bv', 'last', 'rows', 'dim', 'sched', 'step')] + scal
        return a, tabs

    def catch_up(**bad):
        a, tabs = args(**bad)
        return lib.slb_shard_rows_adam_catch_up(a['ids'], a['R'], *tabs, stream)

    def step(**bad):
        a, tabs = args(**bad)
        return lib.slb_shard_rows_adam(a['ids'], a['g'], a['gb'], a['R'], *tabs, a['ws'], a['wsb'], stream)

    before = [x.clone() for x in t]
    common = [dict(ids=None), dict(W=None), dict(m=None), dict(v=None), dict(b=None), dict(bm=None), dict(bv=None),
              dict(last=None), dict(sched=None), dict(R=-1), dict(rows=-3), dict(rows=0), dict(dim=0), dict(step=0),
              dict(step=1 << 31)]
    for bad in common:
        assert catch_up(**bad) != 0, bad
        assert lib.slb_last_error()
    for bad in common + [dict(g=None), dict(gb=None), dict(ws=None), dict(wsb=need - 1)]:
        assert step(**bad) != 0, bad
        assert lib.slb_last_error()
    torch.cuda.synchronize()
    for x, y in zip(t, before):
        assert torch.equal(x, y)
    assert catch_up() == 0 and step() == 0
    torch.cuda.synchronize()
    assert not torch.equal(t[0], before[0])


# ------------------------------------------------------------------ ShardedSeq and fit on NCCL

STEP_JOBS = [('pool', 'pointwise', 1e-2), ('cnn', 'bpr', 0.0), ('lstm', 'adaptive_hinge', 1e-2),
             ('mixture', 'bpr', 1e-2)]
FIT_JOBS = [('pooling', 'bpr'), ('cnn', 'pointwise'), ('lstm', 'pointwise'), ('mixture', 'bpr')]
FIT_OPT = dict(lr=1e-2, weight_decay=1e-3)


def _step_job(rank, world, dev, net, loss, wd):
    from spotlight_b200.optim import fused_adam
    from spotlight_b200.sharded import GpuBackend, SeqShardState, ShardedSeq, ShardPlan, _rank_slice
    I, D, S = tac.STEP['I'], tac.STEP['D'], tac.STEP['S']
    n_neg = tac._n_neg(loss)
    E, bias, lstm, mix, convs = tac.step_params(net, I)
    t = lambda d: None if d is None else {k: (torch.from_numpy(v) if isinstance(v, np.ndarray) else v)   # noqa: E731
                                         for k, v in d.items()}
    plan = ShardPlan(1, I, world)
    st = SeqShardState(plan, rank, D, dev, init=(torch.from_numpy(E), torch.from_numpy(bias)),
                       convs=None if convs is None else [(torch.from_numpy(w), torch.from_numpy(b)) for w, b in convs],
                       lstm=t(lstm), mixture=t(mix), optimizer_func=fused_adam(lr=tac.LR, weight_decay=wd))
    be = GpuBackend(dev)
    model = ShardedSeq(plan, st, rank, be, cnn=tac.CNN if convs is not None else None, n_neg=n_neg)
    losses = []
    for seqs, negs in tac.step_batches(tac.STEP['seed'] + 2, I, S, n_neg):
        B = seqs.shape[0]
        a, c = _rank_slice(B, rank, world)
        mine = negs.reshape(n_neg, B, S)[:, a:c].reshape(-1, S)
        d = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(dev)      # noqa: E731
        losses.append(float(model.step(d(seqs[a:c]), d(mine), loss)))
    be.owner_adam_flush(st)
    return gather_state(st, plan, I), losses, st.last.cpu().numpy(), st.opt.steps_taken


def _fit_job(rank, world, dev, rep, loss):
    from spotlight_b200.interactions import SequenceInteractions
    from spotlight_b200.optim import fused_adam
    from spotlight_b200.sharded import ShardedImplicitSequenceModel
    F = tsg.FIT
    rs = np.random.RandomState(F['seed'])
    model = ShardedImplicitSequenceModel(F['I'], rank, world, dev, loss=loss, representation=rep, embedding_dim=F['D'],
                                         n_iter=F['n_iter'], batch_size=F['B'], random_state=rs,
                                         optimizer_func=fused_adam(**FIT_OPT))
    model.fit(SequenceInteractions(tsg._fit_data(), num_items=F['I']))
    net = model.gathered_net()
    sd = {k: v.detach().cpu().numpy().copy() for k, v in net.state_dict().items()}
    last = model.state.last.cpu().numpy()
    return sd, model.epoch_losses, rs.get_state(), (int(last.min()), int(last.max())), model.state.opt.steps_taken


def _jobs(rank, world, dev):
    res = {}
    for job in STEP_JOBS:
        res['step', job] = _step_job(rank, world, dev, *job)
    if world == 1:
        for rep, loss in FIT_JOBS:
            res['fit', rep, loss] = _fit_job(rank, world, dev, rep, loss)
    return res


_CACHE = {}


def _results(world):
    if torch.cuda.device_count() < world:
        pytest.skip('needs %d GPUs' % world)
    if world not in _CACHE:
        _CACHE[world] = sc.run_world(_jobs, world, backend='nccl', timeout=900)
    return _CACHE[world]


@pytest.mark.parametrize('world', [1, 2])
@pytest.mark.parametrize('net,loss,wd', STEP_JOBS)
def test_sharded_seq_adam_step_gpu_matches_dense_adam(world, net, loss, wd):
    """The CPU test's four steps (ranks without sequences at world 2, one row requested by every
    rank, rows only the flush moves) on the product kernels against whole-minibatch float64 steps
    with dense Adam, after the flush; every row current for the step count."""
    res = _results(world)
    got, losses, _, _ = res[0]['step', (net, loss, wd)]
    I = tac.STEP['I']
    ref, ref_losses = tac.adam_trajectory(net, I, loss, tac._n_neg(loss), wd)
    assert_close(np.array(losses), np.array(ref_losses), 2e-5, what='losses')
    assert len(got) == len(ref)
    for k, (a, b) in enumerate(zip(got, ref)):
        # fp32 gradients on the device: 1e-4 of the scale, a percent of one Adam step
        tac._check_adam(a, b, tac.LR, 'param%d' % k, rtol=1e-4)
    for r in range(world):
        last, steps = res[r]['step', (net, loss, wd)][2:]
        assert steps == len(tac.SIZES) and (last == steps).all()


_SINGLE = {}


def _single_gpu_fit(rep, loss):
    if (rep, loss) not in _SINGLE:
        from spotlight_b200.interactions import SequenceInteractions
        from spotlight_b200.optim import fused_adam
        from spotlight_b200.sequence.implicit import ImplicitSequenceModel
        F = tsg.FIT
        rs = np.random.RandomState(F['seed'])
        one = ImplicitSequenceModel(loss=loss, representation=rep, embedding_dim=F['D'], n_iter=F['n_iter'],
                                    batch_size=F['B'], use_cuda=True, random_state=rs,
                                    optimizer_func=fused_adam(**FIT_OPT))
        buf = io.StringIO()
        with contextlib.redirect_stdout(buf):
            one.fit(SequenceInteractions(tsg._fit_data(), num_items=F['I']), verbose=True)
        assert one._route() == 'fused'
        losses = [float(line.split('loss')[1]) for line in buf.getvalue().splitlines() if line.startswith('Epoch')]
        sd = {k: v.detach().cpu().numpy() for k, v in one._net.state_dict().items()}
        _SINGLE[rep, loss] = (sd, losses, rs.get_state(), one._optimizer.steps_taken)
    return _SINGLE[rep, loss]


@pytest.mark.parametrize('rep,loss', FIT_JOBS)
def test_sharded_sequence_fit_adam_equals_single_gpu_fit(rep, loss):
    """World 1: fit() with fused_adam(lr=1e-2, weight_decay=1e-3) through the whole sharded route
    (bucketing, owner catch-up, all-to-alls with itself, owner Adam, replicated Adam, flush) against
    ImplicitSequenceModel(fused_adam) from the same seed: epoch losses, parameters (the tolerances
    of test_seq_adam_gpu's fused-route fit test), the RandomState position, and every row current
    for the step count."""
    sd, losses, state, (lo, hi), steps = _results(1)[0]['fit', rep, loss]
    want_sd, want_losses, want_state, want_steps = _single_gpu_fit(rep, loss)
    assert len(losses) == tsg.FIT['n_iter']
    assert_close(np.array(losses), np.array(want_losses), 1e-5, what='epoch losses')
    assert sorted(sd) == sorted(want_sd)
    for k in sd:
        assert_close(sd[k], want_sd[k], 5e-4, atol=1e-7, what=k)
    assert np.array_equal(state[1], want_state[1]) and state[2] == want_state[2]
    assert steps == want_steps and lo == hi == steps
