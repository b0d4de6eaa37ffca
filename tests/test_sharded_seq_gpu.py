"""GPU tests of the sharded sequence training on the product kernels: the owner-side row-wise
Adagrad kernel against NumPy float64, ShardedSeq steps of LSTMNet and MixtureLSTMNet against the
float64 oracle (NCCL, world 1 always, world 2 when two GPUs are visible; one process group per
world runs all jobs), and ShardedImplicitSequenceModel.fit() at world 1 against the single-GPU
ImplicitSequenceModel with fused_adagrad on the same data and seed."""

import contextlib
import io
import os
import sys
import types

import numpy as np
import pytest
import torch

from conftest import ROOT, assert_close

sys.path.insert(0, os.path.join(ROOT, 'tests'))
pytestmark = pytest.mark.gpu

import sharded_common as sc                                                       # noqa: E402
from test_sharded_seq_cpu import (gather_state, make_batches, make_params,          # noqa: E402
                                  oracle_trajectory, owner_case, owner_update_reference)

# ------------------------------------------------------------------ owner update kernel


def _state(W, S, b, sb, dev):
    t = lambda x: torch.from_numpy(x.copy()).to(dev)        # noqa: E731
    return types.SimpleNamespace(Wi=t(W), sWi=t(S), bi=t(b), sbi=t(sb), lr=0.05, eps=1e-10)


def _run_owner(case, dev):
    from spotlight_b200.sharded import GpuBackend
    ids, g_rows, g_bias, W, S, b, sb = case
    st = _state(W, S, b, sb, dev)
    GpuBackend(dev).owner_update(st, torch.from_numpy(ids).to(dev), torch.from_numpy(g_rows).to(dev),
                                 torch.from_numpy(g_bias).to(dev))
    torch.cuda.synchronize()
    return [x.cpu().numpy() for x in (st.Wi, st.sWi, st.bi, st.sbi)]


TILES = 3 * 4096 + 17           # rows spanning several of segindex.cuh's 4096-row scan tiles


def _hot_case(seed, rows, D, hot_row=7, peers=(9, 0, 14, 5)):
    """One row requested at 300 positions (more than any lane group's in-register sort holds)."""
    ids, g_rows, g_bias, W, S, b, sb = owner_case(seed, rows, D, peers=peers)
    rs = np.random.RandomState(seed + 1)
    hot = np.full(300, hot_row, dtype=np.int64)
    ids = np.concatenate([ids, hot])
    g_rows = np.concatenate([g_rows, rs.randn(300, D).astype(np.float32)])
    g_bias = np.concatenate([g_bias, rs.randn(300).astype(np.float32)])
    return ids, g_rows, g_bias, W, S, b, sb


@pytest.mark.parametrize('D', [1, 3, 4, 64, 128, 512])
@pytest.mark.parametrize('kind', ['peers', 'padding', 'hot', 'tiles'])
def test_owner_update_kernel_matches_numpy(D, kind):
    """Duplicate ids across peers, an empty peer, -1 padding slots or a hot row ('tiles': over a
    row space of several scan tiles, the hot row just past a tile edge): each distinct row takes one
    Adagrad step on the rank-order sum of its contributions; untouched rows and their states are
    unchanged bit for bit; two runs are bit-identical."""
    dev = torch.device('cuda', 0)
    rows = TILES if kind == 'tiles' else 300
    if kind == 'hot':
        case = _hot_case(5, rows, D)
    elif kind == 'tiles':
        case = _hot_case(5, rows, D, hot_row=4096, peers=(900, 0, 1400, 500))
    else:
        case = owner_case(5, rows, D, peers=(90, 0, 140, 50), padding=5 if kind == 'padding' else 0)
    ids, g_rows, g_bias, W, S, b, sb = case
    want = owner_update_reference(ids, g_rows, g_bias, W, S, b, sb, 0.05)
    got = _run_owner(case, dev)
    for g, w, nm in zip(got, want, ('W', 'state_W', 'b', 'state_b')):
        assert_close(g, w, 1e-5, what=nm)
    untouched = np.setdiff1d(np.arange(rows), ids)
    assert len(untouched) > 0
    for g, x in zip(got, (W, S, b, sb)):
        assert np.array_equal(g[untouched], x[untouched])
    again = _run_owner(case, dev)
    for g, a in zip(got, again):
        assert np.array_equal(g, a)


def test_owner_update_kernel_empty_and_rejections():
    """R == 0 changes nothing (and needs no storage); null pointers, negative sizes, rows for an
    empty shard and a short workspace are rejected before any launch."""
    from spotlight_b200 import _lib, ops
    dev = torch.device('cuda', 0)
    lib = _lib.load()
    ids, g_rows, g_bias, W, S, b, sb = owner_case(2, 50, 8)
    st = _state(W, S, b, sb, dev)
    from spotlight_b200.sharded import GpuBackend
    GpuBackend(dev).owner_update(st, torch.zeros(0, dtype=torch.int64, device=dev),
                                 torch.zeros((0, 8), device=dev), torch.zeros(0, device=dev))
    torch.cuda.synchronize()
    assert np.array_equal(st.Wi.cpu().numpy(), W) and np.array_equal(st.bi.cpu().numpy(), b)
    stream = ops._stream()
    assert lib.slb_shard_rows_adagrad(None, None, None, 0, None, None, None, None, 0, 8, 0.05, 1e-10,
                                      None, 0, stream) == 0
    R, rows = len(ids), 50
    d = {k: torch.from_numpy(v).to(dev) for k, v in (('ids', ids), ('g', g_rows), ('gb', g_bias))}
    need = lib.slb_shard_rows_workspace_bytes(R, rows)
    ws = torch.zeros(need, dtype=torch.uint8, device=dev)
    P = ops._ptr

    def call(ids_p=P(d['ids']), g=P(d['g']), gb=P(d['gb']), n=R, Wp=P(st.Wi), Sp=P(st.sWi), bp=P(st.bi),
             sbp=P(st.sbi), nrows=rows, dim=8, wsp=P(ws), wsb=need):
        return lib.slb_shard_rows_adagrad(ids_p, g, gb, n, Wp, Sp, bp, sbp, nrows, dim, 0.05, 1e-10, wsp, wsb, stream)

    before = [x.clone() for x in (st.Wi, st.sWi, st.bi, st.sbi)]
    for bad in (dict(ids_p=None), dict(g=None), dict(gb=None), dict(Wp=None), dict(Sp=None), dict(bp=None),
                dict(sbp=None), dict(wsp=None), dict(n=-1), dict(nrows=-3), dict(dim=0), dict(dim=-4),
                dict(nrows=0)):
        assert call(**bad) != 0, bad
        assert lib.slb_last_error()
    assert call(wsb=need - 1) != 0
    torch.cuda.synchronize()
    for x, y in zip((st.Wi, st.sWi, st.bi, st.sbi), before):
        assert torch.equal(x, y)
    assert call() == 0
    torch.cuda.synchronize()
    assert not torch.equal(st.Wi, before[0])


# ------------------------------------------------------------------ ShardedSeq and fit on NCCL

STEP = dict(seed=13, I=300, D=32, B=24, S=20, steps=3)
STEP_JOBS = [('lstm', 'bpr'), ('mixture', 'pointwise')]

FIT = dict(seed=29, I=1500, D=32, S=20, n=700, B=128, n_iter=2)
FIT_JOBS = [('pooling', 'bpr'), ('cnn', 'pointwise'), ('lstm', 'pointwise'), ('mixture', 'bpr')]


def _fit_data():
    rs = np.random.RandomState(FIT['seed'] + 3)
    seqs = rs.randint(1, FIT['I'], (FIT['n'], FIT['S'])).astype(np.int64)
    for b in range(FIT['n']):
        seqs[b, :rs.randint(0, FIT['S'])] = 0
    return seqs


def _step_job(rank, world, dev, net, loss):
    from spotlight_b200.sharded import GpuBackend, SeqShardState, ShardedSeq, ShardPlan, _rank_slice
    E, bias, lstm, mix = make_params(STEP['seed'], STEP['I'], STEP['D'], net)
    batches = make_batches(STEP['seed'] + 2, STEP['I'], STEP['B'], STEP['S'], STEP['steps'], 1)
    t = lambda d: None if d is None else {k: (torch.from_numpy(v) if isinstance(v, np.ndarray) else v)   # noqa: E731
                                         for k, v in d.items()}
    plan = ShardPlan(1, STEP['I'], world)
    st = SeqShardState(plan, rank, STEP['D'], dev, lr=0.05, init=(torch.from_numpy(E), torch.from_numpy(bias)),
                       lstm=t(lstm), mixture=t(mix))
    model = ShardedSeq(plan, st, rank, GpuBackend(dev))
    losses = []
    for seqs, negs in batches:
        a, c = _rank_slice(seqs.shape[0], rank, world)
        d = lambda x: torch.from_numpy(np.ascontiguousarray(x[a:c])).to(dev)      # noqa: E731
        losses.append(float(model.step(d(seqs), d(negs), loss)))
    return gather_state(st, plan, STEP['I']), losses


def _fit_job(rank, world, dev, rep, loss):
    from spotlight_b200.interactions import SequenceInteractions
    from spotlight_b200.sharded import ShardedImplicitSequenceModel
    rs = np.random.RandomState(FIT['seed'])
    model = ShardedImplicitSequenceModel(FIT['I'], rank, world, dev, loss=loss, representation=rep,
                                         embedding_dim=FIT['D'], n_iter=FIT['n_iter'], batch_size=FIT['B'],
                                         learning_rate=0.05, random_state=rs)
    model.fit(SequenceInteractions(_fit_data(), num_items=FIT['I']))
    net = model.gathered_net()
    sd = {k: v.detach().cpu().numpy().copy() for k, v in net.state_dict().items()}
    return sd, model.epoch_losses, rs.get_state()


def _jobs(rank, world, dev):
    res = {}
    for net, loss in STEP_JOBS:
        res['step', net, loss] = _step_job(rank, world, dev, net, loss)
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
@pytest.mark.parametrize('net,loss', STEP_JOBS)
def test_sharded_seq_step_gpu_matches_oracle(world, net, loss):
    got, losses = _results(world)[0]['step', net, loss]
    params = make_params(STEP['seed'], STEP['I'], STEP['D'], net)
    batches = make_batches(STEP['seed'] + 2, STEP['I'], STEP['B'], STEP['S'], STEP['steps'], 1)
    ref, ref_losses = oracle_trajectory(params, batches, loss, 0.05, 1)
    assert_close(np.array(losses), np.array(ref_losses), 2e-5, what='losses')
    assert len(got) == len(ref)
    for k, (a, b) in enumerate(zip(got, ref)):
        # Adagrad trajectory tolerance, as test_sharded_gpu's sequence case: first-touch
        # normalisation amplifies 1e-7 gradient differences on near-cancelling rows
        assert_close(a, b.reshape(a.shape), 5e-3, what='param%d' % k)


_SINGLE = {}


def _single_gpu_fit(rep, loss):
    if (rep, loss) not in _SINGLE:
        from spotlight_b200.interactions import SequenceInteractions
        from spotlight_b200.optim import fused_adagrad
        from spotlight_b200.sequence.implicit import ImplicitSequenceModel
        rs = np.random.RandomState(FIT['seed'])
        one = ImplicitSequenceModel(loss=loss, representation=rep, embedding_dim=FIT['D'], n_iter=FIT['n_iter'],
                                    batch_size=FIT['B'], use_cuda=True, random_state=rs,
                                    optimizer_func=fused_adagrad(lr=0.05))
        buf = io.StringIO()
        with contextlib.redirect_stdout(buf):
            one.fit(SequenceInteractions(_fit_data(), num_items=FIT['I']), verbose=True)
        assert one._route() == 'fused'
        losses = [float(line.split('loss')[1]) for line in buf.getvalue().splitlines() if line.startswith('Epoch')]
        sd = {k: v.detach().cpu().numpy() for k, v in one._net.state_dict().items()}
        _SINGLE[rep, loss] = (sd, losses, rs.get_state())
    return _SINGLE[rep, loss]


@pytest.mark.parametrize('rep,loss', FIT_JOBS)
def test_sharded_sequence_fit_equals_single_gpu_fit(rep, loss):
    """World 1: the estimator's whole sharded route (bucketing, all-to-alls with itself, owner
    update, replicated-parameter all-reduce) against ImplicitSequenceModel(fused_adagrad) from the
    same seed: the same starting weights, minibatches and negatives give the same epoch losses
    and parameters (the tolerances of the single-GPU fused_adagrad fit test) and leave the
    RandomState at the same position."""
    sd, losses, state = _results(1)[0]['fit', rep, loss]
    want_sd, want_losses, want_state = _single_gpu_fit(rep, loss)
    assert len(losses) == FIT['n_iter']
    assert_close(np.array(losses), np.array(want_losses), 1e-5, what='epoch losses')
    assert sorted(sd) == sorted(want_sd)
    for k in sd:
        assert_close(sd[k], want_sd[k], 1e-4, atol=1e-7, what=k)
    assert np.array_equal(state[1], want_state[1]) and state[2] == want_state[2]
