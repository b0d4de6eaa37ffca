"""World-size-2 and 3 gloo tests of sharded sequence training with row-wise lazy-exact Adam
(``optimizer_func=fused_adam``) on CPU, with a NumPy backend whose owner-side Adam is
oracle.adam.LazyAdamTable in float64: ShardedSeq steps of PoolNet, CNNNet, LSTMNet and
MixtureLSTMNet against the single-process float64 oracle with dense Adam on every row, and
ShardedImplicitSequenceModel.fit() against a float64 replay of the reference's stream.  Also the
optimizer selection and the resource usage of the owner-side Adam kernels."""

import os
import sys

import numpy as np
import pytest
import torch

from conftest import ROOT, assert_close

sys.path.insert(0, os.path.join(ROOT, 'tests'))

import sharded_common as sc            # noqa: E402
import test_sharded_seq_cpu as tsc     # noqa: E402
from oracle.adam import LazyAdamTable  # noqa: E402

LR = 1e-2


class AdamSeqBackend(tsc.SeqBackend):
    """SeqBackend plus the owner-side lazy-exact Adam, in float64 on the float32 shard and state
    tensors of SeqShardState."""

    @staticmethod
    def _tables(st):
        hp = st.opt.fused_hparams()
        kw = dict(lr=hp['lr'], betas=(hp['beta1'], hp['beta2']), eps=hp['eps'], weight_decay=hp['weight_decay'])
        tabs = []
        for w, m, v in ((st.Wi, st.mWi, st.vWi), (st.bi, st.mbi, st.vbi)):
            tab = LazyAdamTable(w.numpy(), **kw)
            tab.m = m.numpy().astype(np.float64).reshape(tab.w.shape)
            tab.v = v.numpy().astype(np.float64).reshape(tab.w.shape)
            tab.last = st.last.numpy().astype(np.int64)         # the row and its bias share `last`
            tabs.append(tab)
        return tabs

    @staticmethod
    def _store(st, tabs):
        for tab, tensors in zip(tabs, ((st.Wi, st.mWi, st.vWi), (st.bi, st.mbi, st.vbi))):
            for dst, src in zip(tensors, (tab.w, tab.m, tab.v)):
                dst.copy_(torch.from_numpy(src.reshape(dst.shape).astype(np.float32)))
        assert np.array_equal(tabs[0].last, tabs[1].last)
        st.last.copy_(torch.from_numpy(tabs[0].last.astype(np.int32)))

    @staticmethod
    def _in_range(st, local_ids):
        ids = local_ids.numpy()
        return ids[(ids >= 0) & (ids < st.Wi.shape[0])]

    def owner_adam_catch_up(self, st, local_ids, t):
        ids = self._in_range(st, local_ids)
        if len(ids):
            tabs = self._tables(st)
            for tab in tabs:
                tab.catch_up(ids, t - 1)
            self._store(st, tabs)

    def owner_adam_update(self, st, local_ids, g_rows, g_bias, t):
        ids = local_ids.numpy()
        keep = (ids >= 0) & (ids < st.Wi.shape[0])
        if not keep.any():
            return
        rows = np.unique(ids[keep])
        slot = np.searchsorted(rows, ids[keep])
        dW = np.zeros((len(rows), st.Wi.shape[1]))
        db = np.zeros(len(rows))
        np.add.at(dW, slot, g_rows.numpy()[keep].astype(np.float64))       # position (= rank) order
        np.add.at(db, slot, g_bias.numpy().reshape(-1)[keep].astype(np.float64))
        tabs = self._tables(st)
        tabs[0].apply(rows, dW, t)
        tabs[1].apply(rows, db, t)
        self._store(st, tabs)

    def owner_adam_flush(self, st):
        if st.Wi.shape[0]:
            tabs = self._tables(st)
            for tab in tabs:
                tab.flush(st.opt.steps_taken)
            self._store(st, tabs)


class DenseAdam(object):
    """torch.optim.Adam in float64 on a list of arrays: every element moves at every step."""

    def __init__(self, lr, weight_decay, betas=(0.9, 0.999), eps=1e-8):
        self.lr, self.wd, (self.b1, self.b2), self.eps = lr, weight_decay, betas, eps
        self.t, self.m, self.v = 0, None, None

    def __call__(self, P, grads, store=None):
        """One step on P with ``grads``; ``store`` rounds the parameters to that storage type."""
        if self.m is None:
            self.m, self.v = [np.zeros_like(p) for p in P], [np.zeros_like(p) for p in P]
        self.t += 1
        ss, bc = self.lr / (1.0 - self.b1 ** self.t), np.sqrt(1.0 - self.b2 ** self.t)
        for k, g in enumerate(grads):
            g = g.reshape(P[k].shape) + self.wd * P[k]
            self.m[k] += (g - self.m[k]) * (1.0 - self.b1)
            self.v[k] = self.v[k] * self.b2 + (1.0 - self.b2) * g * g
            P[k] -= ss * (self.m[k] / (np.sqrt(self.v[k]) / bc + self.eps))
            if store is not None:
                P[k][...] = P[k].astype(store)


# ------------------------------------------------------------------ ShardedSeq steps

STEP = dict(seed=21, I=41, D=8, S=7)
SIZES = (10, 1, 9, 2)        # minibatch sizes: 1 and 2 leave ranks without sequences at worlds 2 and 3
SHARED = 5                   # an item in every sequence: requested by every rank with sequences
CNN = dict(kernel_width=[3], dilation=[1], nonlinearity='tanh', residual=True)


def _pool(I):
    """Items the minibatches draw: [14, 28) is never drawn at I = 41, the whole item range of rank 1
    at world 3, so only the flush moves those rows."""
    return np.r_[1:14, 28:I] if I > 28 else np.arange(1, I)


def step_batches(seed, I, S, n_neg):
    rs = np.random.RandomState(seed)
    pool = _pool(I)
    out = []
    for B in SIZES:
        seqs = rs.choice(pool, (B, S)).astype(np.int64)
        for b in range(B):
            seqs[b, :rs.randint(0, S)] = 0
        seqs[:, -1] = min(SHARED, I - 1)
        negs = rs.choice(np.r_[0, pool], (n_neg * B, S)).astype(np.int64)
        out.append((seqs, negs))
    return out


def step_params(net, I):
    E, bias, lstm, mix = tsc.make_params(STEP['seed'], I, STEP['D'], net)
    convs = None
    if net == 'cnn':
        rs = np.random.RandomState(STEP['seed'] + 3)
        D = STEP['D']
        convs = [((rs.randn(D, D, 3, 1) * 0.2).astype(np.float32), (rs.randn(D) * 0.1).astype(np.float32))]
    return E, bias, lstm, mix, convs


def adam_trajectory(net, I, loss, n_neg, wd):
    """Single process: whole-minibatch float64 oracle steps + dense Adam on every parameter."""
    E, bias, lstm, mix, convs = step_params(net, I)
    P = [E.astype(np.float64), bias.astype(np.float64)]
    if convs is not None:
        P += [x.astype(np.float64) for wb in convs for x in wb]
    if lstm is not None:
        P += [lstm[k].astype(np.float64) for k in tsc.LSTM_KEYS]
    if mix is not None:
        P += [mix['w'].astype(np.float64), mix['b'].astype(np.float64)]
    adam = DenseAdam(LR, wd)
    losses = []
    for seqs, negs in step_batches(STEP['seed'] + 2, I, STEP['S'], n_neg):
        k = 2
        cv = None
        if convs is not None:
            cv, k = [(P[2], P[3])], 4
        lp = dict(zip(tsc.LSTM_KEYS, P[k:k + 4])) if lstm is not None else None
        mp_ = dict(w=P[k + 4], b=P[k + 5], num_mixtures=mix['num_mixtures']) if mix is not None else None
        r, grads = tsc.oracle_seq_step(P[0], P[1], lp, mp_, seqs, negs, loss, n_neg, cv,
                                       CNN if convs is not None else None)
        losses.append(float(r['loss']))
        adam(P, [r['dE'], r['dbias']] + grads)
    return P, losses


STEP_JOBS = [(net, loss, wd, 41) for net in ('pool', 'cnn', 'lstm', 'mixture')
             for loss in ('pointwise', 'bpr', 'adaptive_hinge') for wd in (0.0, 1e-2)]
STEP_JOBS += [('pool', 'bpr', 1e-2, 4)]        # I = 4 at world 3: rank 2 has an empty item range


def _n_neg(loss):
    return 3 if loss == 'adaptive_hinge' else 1


def _step_job(rank, world, net, loss, wd, I):
    from spotlight_b200.optim import fused_adam
    from spotlight_b200.sharded import SeqShardState, ShardedSeq, ShardPlan, _rank_slice
    n_neg = _n_neg(loss)
    E, bias, lstm, mix, convs = step_params(net, I)
    t = lambda d: None if d is None else {k: (torch.from_numpy(v) if isinstance(v, np.ndarray) else v)   # noqa: E731
                                         for k, v in d.items()}
    plan = ShardPlan(1, I, world)
    st = SeqShardState(plan, rank, STEP['D'], 'cpu', init=(torch.from_numpy(E), torch.from_numpy(bias)),
                       convs=None if convs is None else [(torch.from_numpy(w), torch.from_numpy(b)) for w, b in convs],
                       lstm=t(lstm), mixture=t(mix), optimizer_func=fused_adam(lr=LR, weight_decay=wd))
    be = AdamSeqBackend()
    model = ShardedSeq(plan, st, rank, be, cnn=CNN if convs is not None else None, n_neg=n_neg)
    losses = []
    for seqs, negs in step_batches(STEP['seed'] + 2, I, STEP['S'], n_neg):
        B, S = seqs.shape
        a, c = _rank_slice(B, rank, world)
        mine = negs.reshape(n_neg, B, S)[:, a:c].reshape(-1, S)
        losses.append(float(model.step(torch.from_numpy(seqs[a:c].copy()), torch.from_numpy(mine.copy()), loss)))
    be.owner_adam_flush(st)
    return tsc.gather_state(st, plan, I), losses, st.last.numpy().copy(), st.opt.steps_taken


def _step_jobs(rank, world, dev):
    return {job: _step_job(rank, world, *job) for job in STEP_JOBS}


_CACHE = {}


def _step_results(world):
    if world not in _CACHE:
        _CACHE[world] = sc.run_world(_step_jobs, world)
    return _CACHE[world]


def _check_adam(got, want, lr, what, rtol=1e-5):
    """Parameters after Adam steps: ``rtol`` of their scale, or for a few elements (2 %, at least
    two) a tenth of a step, where a gradient component sits at the fp32 rounding level of its
    minibatch sum (the sharded route adds the
    ranks' fp32 partial gradients; Adam's first step moves such a component by lr * g / |g|)."""
    err = np.abs(got.astype(np.float64) - want.reshape(got.shape))
    tol = np.maximum(rtol * np.abs(want).max(), 1e-7)
    bad = err > tol
    assert err.max() <= 0.1 * lr, '%s: max error %.3e' % (what, err.max())
    assert bad.sum() <= max(2, 0.02 * bad.size), '%s: %d of %d elements off by more than %.1e' % (
        what, bad.sum(), bad.size, tol)


@pytest.mark.parametrize('world', [2, 3])
@pytest.mark.parametrize('net,loss,wd,I', STEP_JOBS)
def test_sharded_seq_adam_step_matches_dense_adam(world, net, loss, wd, I):
    """Four steps with minibatches of 10, 1, 9 and 2 sequences (ranks without sequences at both
    worlds), one item in every sequence (the same row requested by every rank) and an item range
    no minibatch draws; after the final flush, the gathered table, bias and replicated parameters
    equal whole-minibatch float64 steps with dense Adam on every row at every step, and every row
    of every rank is current for the step count."""
    if I == 4 and world != 3:
        pytest.skip('the empty item range arises at world 3')
    res = _step_results(world)
    got, losses, _, _ = res[0][net, loss, wd, I]
    ref, ref_losses = adam_trajectory(net, I, loss, _n_neg(loss), wd)
    assert_close(np.array(losses), np.array(ref_losses), 1e-5, what='losses')
    assert len(got) == len(ref)
    for k, (a, b) in enumerate(zip(got, ref)):
        _check_adam(a, b, LR, 'param%d' % k)
    for r in range(world):
        assert res[r][net, loss, wd, I][1] == losses
        last, steps = res[r][net, loss, wd, I][2:]
        assert steps == len(SIZES) and (last == steps).all()
    if I == 4:
        assert res[2][net, loss, wd, I][2].size == 0
    if I == 41 and wd > 0:
        E0 = step_params(net, I)[0]
        assert not np.array_equal(got[0][14:28], E0[14:28])      # moved by the flush alone


# ------------------------------------------------------------------ ShardedImplicitSequenceModel.fit

FIT_JOBS = [('pooling', 'pointwise'), ('cnn', 'bpr'), ('lstm', 'adaptive_hinge'), ('mixture', 'pointwise')]
WD = 1e-3


def _fit_job(rank, world, rep, loss, splits):
    from spotlight_b200.interactions import SequenceInteractions
    from spotlight_b200.optim import fused_adam
    from spotlight_b200.sharded import ShardedImplicitSequenceModel
    rs = np.random.RandomState(tsc.FIT['seed'])
    model = ShardedImplicitSequenceModel(tsc.FIT['I'], rank, world, 'cpu', loss=loss, representation=rep,
                                         embedding_dim=tsc.FIT['D'], n_iter=tsc.FIT['n_iter'] // splits,
                                         batch_size=tsc.FIT['B'], random_state=rs, num_negative_samples=3,
                                         backend=AdamSeqBackend(), optimizer_func=fused_adam(lr=LR, weight_decay=WD))
    inter = SequenceInteractions(tsc._fit_data(), num_items=tsc.FIT['I'])
    for _ in range(splits):
        model.fit(inter)
    net = model.gathered_net()
    params = [p.detach().numpy().copy() for p in net.parameters()]
    return params, model.epoch_losses, rs.get_state(), model.state.opt.steps_taken


def _fit_jobs(rank, world, dev):
    return {(rep, loss, splits): _fit_job(rank, world, rep, loss, splits)
            for rep, loss in FIT_JOBS for splits in (1, 2)}


_FIT = {}


def _fit_results():
    if not _FIT:
        _FIT.update(sc.run_world(_fit_jobs, 2))
    return _FIT


def _replay(rep, loss, n_neg, calls, store=None):
    """The single-process fit() called ``calls`` times for FIT['n_iter'] epochs in all: the
    constructor's draw and set_seed, the net built as _initialize builds it, each call restarting
    from the interactions' order, per epoch one cumulative shuffle and one (n_seq * n_neg, S) draw,
    minibatches of B rows stepped whole through the float64 oracle, and dense Adam (weight decay
    included) on every parameter, its step count and moments carried across calls."""
    from spotlight_b200.sequence.representations import CNNNet, LSTMNet, MixtureLSTMNet, PoolNet
    from spotlight_b200.torch_utils import set_seed
    F = tsc.FIT
    rs = np.random.RandomState(F['seed'])
    set_seed(rs.randint(-10 ** 8, 10 ** 8))
    net = {'pooling': PoolNet, 'cnn': CNNNet, 'lstm': LSTMNet, 'mixture': MixtureLSTMNet}[rep](F['I'], F['D'])
    names = [nm for nm, _ in net.named_parameters()]
    P = [p.detach().numpy().astype(np.float64).copy() for p in net.parameters()]
    by = dict(zip(names, P))
    lstm_names = dict(zip(tsc.LSTM_KEYS, ('weight_ih', 'weight_hh', 'bias_ih', 'bias_hh')))
    adam = DenseAdam(LR, WD)
    n, S, B = F['n'], F['S'], F['B']
    epoch_losses = []
    for _ in range(calls):
        seqs = tsc._fit_data()
        for _ in range(F['n_iter'] // calls):
            order = np.arange(n)
            rs.shuffle(order)
            seqs = seqs[order]
            negatives = rs.randint(0, F['I'], (n * n_neg, S), dtype=np.int64)
            losses = []
            for lo in range(0, n, B):
                m = min(B, n - lo)
                lstm = mix = convs = cnn = None
                if 'lstm.weight_ih_l0' in by:
                    lstm = {k: by['lstm.%s_l0' % nm] for k, nm in lstm_names.items()}
                if 'projection.weight' in by:
                    mix = dict(w=by['projection.weight'], b=by['projection.bias'], num_mixtures=net.num_mixtures)
                if rep == 'cnn':
                    cnn = dict(kernel_width=list(net.kernel_width), dilation=list(net.dilation), nonlinearity='tanh',
                               residual=True)
                    convs = [(by['cnn_%d.weight' % i], by['cnn_%d.bias' % i]) for i in range(len(net.cnn_layers))]
                r, grads = tsc.oracle_seq_step(by['item_embeddings.weight'], by['item_biases.weight'], lstm, mix,
                                               seqs[lo:lo + m], negatives[lo * n_neg:(lo + m) * n_neg], loss, n_neg,
                                               convs, cnn)
                losses.append(float(r['loss']))
                g = {'item_embeddings.weight': r['dE'], 'item_biases.weight': r['dbias']}
                if cnn is not None:
                    for i in range(len(net.cnn_layers)):
                        g['cnn_%d.weight' % i], g['cnn_%d.bias' % i] = grads[2 * i], grads[2 * i + 1]
                if lstm is not None:
                    for k, nm in lstm_names.items():
                        g['lstm.%s_l0' % nm] = r['dlstm'][k]
                if mix is not None:
                    g['projection.weight'], g['projection.bias'] = r['dmix']['w'], r['dmix']['b']
                adam(P, [g[nm] for nm in names], store=store)
            epoch_losses.append(float(np.mean(losses)))
    return P, epoch_losses, rs, adam.t


@pytest.mark.parametrize('rep,loss', FIT_JOBS)
def test_sharded_sequence_fit_adam_is_the_single_process_fit(rep, loss):
    """fit() at world 2 with fused_adam(weight_decay=1e-3) over two epochs of 47 sequences in
    minibatches of 9 (the last has 2) against the single-process replay of the reference's stream
    with dense float64 Adam; and two fit(n_iter=1) calls against the replay of two calls, which
    resume the step count, the moments and `last`.  Epoch losses, item table, bias, replicated
    parameters, the step count and every rank's final RandomState."""
    n_neg = 3 if loss == 'adaptive_hinge' else 1
    # float32 parameter storage for the hinge, whose kink and argmax over negatives turn the gap
    # between float64 and float32 storage into different active terms (test_sharded_seq_cpu)
    store = np.float32 if loss == 'adaptive_hinge' else None
    res = _fit_results()
    for calls in (1, 2):
        ref, ref_losses, rs, steps = _replay(rep, loss, n_neg, calls, store)
        want = rs.get_state()
        for r in range(2):
            got, losses, state, taken = res[r][rep, loss, calls]
            assert_close(np.array(losses), np.array(ref_losses), 1e-5, what='epoch losses')
            assert len(got) == len(ref)
            for k, (a, b) in enumerate(zip(got, ref)):
                _check_adam(a, b, LR, 'param%d' % k)
            assert np.array_equal(state[1], want[1]) and state[2] == want[2]
            assert taken == steps == tsc.FIT['n_iter'] * -(-tsc.FIT['n'] // tsc.FIT['B'])


# ------------------------------------------------------------------ optimizer selection

def test_sharded_sequence_model_optimizer_selection():
    """None keeps the row-wise Adagrad state at learning_rate; fused_adagrad without weight decay is
    Adagrad with its hyper-parameters; fused_adam builds a FusedAdam over the shard, the bias view
    and the replicated parameters; torch.optim.Adam, fused_sgd and fused_adagrad with weight decay
    are rejected."""
    from spotlight_b200.optim import FusedAdam, fused_adagrad, fused_adam, fused_sgd
    from spotlight_b200.sharded import ShardedImplicitSequenceModel

    def make(func, rep='lstm'):
        return ShardedImplicitSequenceModel(20, 0, 1, 'cpu', representation=rep, embedding_dim=8, learning_rate=0.03,
                                            backend=AdamSeqBackend(), optimizer_func=func)

    st = make(None).state
    assert st.opt is None and (st.lr, st.eps) == (0.03, 1e-10)
    assert st.sWi.shape == st.Wi.shape and st.sbi.shape == st.bi.shape and not st.sWi.any()
    assert all(s is not None and s.shape == p.shape and not s.any() for p, s in st.replicated())
    st = make(fused_adagrad(lr=0.2, eps=1e-6)).state
    assert st.opt is None and (st.lr, st.eps) == (0.2, 1e-6) and st.sWi.shape == st.Wi.shape
    st = make(fused_adam(lr=1e-3, weight_decay=1e-4)).state
    assert isinstance(st.opt, FusedAdam) and st.sWi is None
    assert st.bi2.data_ptr() == st.bi.data_ptr() and st.bi2.shape == (20, 1)
    params = st.opt.param_groups[0]['params']
    assert params[0] is st.Wi and params[1] is st.bi2 and len(params) == 2 + 4
    assert st.mWi.shape == st.Wi.shape and st.last.shape == (20,) and st.mbi.shape == (20, 1)
    for func in (lambda p: torch.optim.Adam(p, lr=1e-3), fused_sgd(lr=0.1), fused_adagrad(lr=0.1, weight_decay=1e-3)):
        with pytest.raises(ValueError, match='fused_adam'):
            make(func)


# ------------------------------------------------------------------ resource usage

def test_owner_adam_kernels_do_not_spill():
    """Every instantiation of rows_adam_catch_up_kernel and rows_adam_kernel (lanes per row 1 .. 32,
    float4 and scalar rows) has no stack frame and no local memory in the built library."""
    from test_mf_resource_usage_cpu import _find, _usage
    usage = _usage()
    for name in ('rows_adam_catch_up_kernel', 'rows_adam_kernel'):
        for lpr in (1, 2, 4, 8, 16, 32):
            for vec in (0, 1):
                r = _find(usage, '%d%sILi%dELb%dEE' % (len(name), name, lpr, vec))
                assert r['STACK'] == 0 and r['LOCAL'] == 0, '%s<%d,%d> spills: %s' % (name, lpr, vec, r)
