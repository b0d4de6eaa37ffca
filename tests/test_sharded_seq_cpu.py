"""World-size-2 and 3 gloo tests of the sharded sequence training on CPU, with a NumPy backend:
ShardedSeq for LSTMNet, MixtureLSTMNet and adaptive hinge, and ShardedImplicitSequenceModel.fit()
against a single-process float64 replay of the reference's minibatch stream.  Also the semantics
of the owner-side row-wise update, and the resource usage of its kernel."""

import os
import sys

import numpy as np
import pytest
import torch

from conftest import ROOT, assert_close

sys.path.insert(0, os.path.join(ROOT, 'tests'))

import sharded_common as sc            # noqa: E402
from oracle import lstm as olstm       # noqa: E402
from oracle import mixture as omix     # noqa: E402
from oracle import seq as oseq         # noqa: E402

LSTM_KEYS = ('w_ih', 'w_hh', 'b_ih', 'b_hh')


def _f64(d):
    return {k: (v.numpy() if torch.is_tensor(v) else v).astype(np.float64) for k, v in d.items() if k != 'num_mixtures'}


def oracle_seq_step(E, bias, lstm, mix, seqs, negs, loss, n_neg, convs=None, cnn=None):
    """The float64 oracle step of one (whole) minibatch; (result, replicated-parameter grads)."""
    if mix is not None:
        r = omix.mixture_step(E, bias, lstm, mix, seqs, negs, mix['num_mixtures'], loss, n_neg, np.float64)
        return r, [r['dlstm'][k] for k in LSTM_KEYS] + [r['dmix']['w'], r['dmix']['b']]
    if lstm is not None:
        r = olstm.lstm_step(E, bias, lstm, seqs, negs, loss, n_neg, np.float64)
        return r, [r['dlstm'][k] for k in LSTM_KEYS]
    if cnn is not None:
        r = oseq.cnn_step(E, bias, convs, seqs, negs, cnn['kernel_width'], cnn['dilation'], loss, n_neg,
                          cnn['nonlinearity'], cnn['residual'], np.float64)
        return r, [x for wb in r['dconvs'] for x in wb]
    r = oseq.pool_step(E, bias, seqs, negs, loss, n_neg, np.float64)
    return r, []


class SeqBackend(sc.NumpyBackend):
    """NumpyBackend plus the LSTMNet / MixtureLSTMNet / n_neg arguments of the sequence step."""

    def seq_local_step(self, E_cache, bias_cache, n_cache, seqs_idx, negs_idx, loss, cnn, norm_count,
                       lstm=None, mixture=None, n_neg=1):
        E = E_cache.numpy().astype(np.float64)
        b = bias_cache.numpy().astype(np.float64).reshape(-1, 1)
        sq, ng = seqs_idx.numpy(), negs_idx.numpy()
        convs = None
        if cnn is not None:
            convs = [(w.numpy().astype(np.float64), c.numpy().astype(np.float64))
                     for w, c in zip(cnn['weights'], cnn['biases'])]
        mix = None
        if mixture is not None:
            mix = dict(_f64(mixture), num_mixtures=int(mixture['num_mixtures']))
        r, grads = oracle_seq_step(E, b, None if lstm is None else _f64(lstm), mix, sq, ng, loss, n_neg,
                                   convs, cnn)
        scale = float((sq != 0).sum()) / float(norm_count.item())
        f = lambda x: torch.from_numpy((x * scale).astype(np.float32))      # noqa: E731
        dconv = [f(g) for g in grads] if cnn is not None else []
        dlstm = {k: f(r['dlstm'][k]) for k in LSTM_KEYS} if lstm is not None else None
        dmix = {k: f(r['dmix'][k]) for k in ('w', 'b')} if mixture is not None else None
        return (torch.tensor(float(r['loss']) * scale, dtype=torch.float32), f(r['dE'])[:n_cache],
                f(r['dbias'].reshape(-1))[:n_cache], dconv[0::2], dconv[1::2], dlstm, dmix)


def make_params(seed, I, D, net, M=2):
    (E, bias, _), _ = sc.make_seq_problem(seed, I, D, 1, 1, 0)
    rs = np.random.RandomState(seed + 1)
    lstm = mix = None
    if net in ('lstm', 'mixture'):
        lstm = {k: (rs.randn(4 * D, D) * 0.3 if k.startswith('w') else rs.randn(4 * D) * 0.1).astype(np.float32)
                for k in LSTM_KEYS}
    if net == 'mixture':
        mix = dict(num_mixtures=M, w=(rs.randn(2 * M * D, D, 1) * 0.3).astype(np.float32),
                   b=(rs.randn(2 * M * D) * 0.1).astype(np.float32))
    return E, bias, lstm, mix


def make_batches(seed, I, B, S, steps, n_neg):
    rs = np.random.RandomState(seed)
    out = []
    for _ in range(steps):
        seqs = rs.randint(1, I, (B, S)).astype(np.int64)
        for b in range(B):
            seqs[b, :rs.randint(0, S)] = 0
        out.append((seqs, rs.randint(0, I, (n_neg * B, S)).astype(np.int64)))
    return out


def adagrad(P, St, grads, lr, eps=1e-10, store=None):
    """Dense Adagrad in float64; ``store`` rounds parameters and states to that storage type."""
    for k, g in enumerate(grads):
        g = g.reshape(P[k].shape)
        St[k] += g * g
        P[k] -= lr * g / (np.sqrt(St[k]) + eps)
        if store is not None:
            P[k][...] = P[k].astype(store)
            St[k][...] = St[k].astype(store)


def oracle_trajectory(params, batches, loss, lr, n_neg):
    """Single process: whole-minibatch float64 oracle steps + dense Adagrad."""
    E, bias, lstm, mix = params
    P = [E.astype(np.float64), bias.astype(np.float64)]
    if lstm is not None:
        P += [lstm[k].astype(np.float64) for k in LSTM_KEYS]
    if mix is not None:
        P += [mix['w'].astype(np.float64), mix['b'].astype(np.float64)]
    St = [np.zeros_like(p) for p in P]
    losses = []
    for seqs, negs in batches:
        lp = dict(zip(LSTM_KEYS, P[2:6])) if lstm is not None else None
        mp_ = dict(w=P[6], b=P[7], num_mixtures=mix['num_mixtures']) if mix is not None else None
        r, grads = oracle_seq_step(P[0], P[1], lp, mp_, seqs, negs, loss, n_neg)
        losses.append(float(r['loss']))
        adagrad(P, St, [r['dE'], r['dbias']] + grads, lr)
    return P, losses


def gather_state(st, plan, I):
    """The full item table and bias of a SeqShardState, then its replicated parameters."""
    out = [sc.gather_rows(st.Wi, plan.ichunk, I), sc.gather_rows(st.bi.reshape(-1, 1), plan.ichunk, I)]
    return out + [p.cpu().numpy() for p, _ in st.replicated()]


# ------------------------------------------------------------------ ShardedSeq steps

STEP = dict(seed=9, I=41, D=8, B=10, S=7, steps=3)
STEP_CASES = [(2, 'lstm', 'bpr', 1), (3, 'lstm', 'pointwise', 1), (2, 'mixture', 'pointwise', 1),
              (3, 'mixture', 'bpr', 1), (2, 'pool', 'adaptive_hinge', 3), (3, 'lstm', 'adaptive_hinge', 2)]


def _step_job(rank, world, dev, net, loss, n_neg):
    from spotlight_b200.sharded import SeqShardState, ShardedSeq, ShardPlan, _rank_slice
    E, bias, lstm, mix = make_params(STEP['seed'], STEP['I'], STEP['D'], net)
    batches = make_batches(STEP['seed'] + 2, STEP['I'], STEP['B'], STEP['S'], STEP['steps'], n_neg)
    t = lambda d: None if d is None else {k: (torch.from_numpy(v) if isinstance(v, np.ndarray) else v)   # noqa: E731
                                         for k, v in d.items()}
    plan = ShardPlan(1, STEP['I'], world)
    st = SeqShardState(plan, rank, STEP['D'], dev, lr=0.05, init=(torch.from_numpy(E), torch.from_numpy(bias)),
                       lstm=t(lstm), mixture=t(mix))
    model = ShardedSeq(plan, st, rank, SeqBackend(), n_neg=n_neg)
    losses = []
    for seqs, negs in batches:
        B, S = seqs.shape
        a, c = _rank_slice(B, rank, world)
        mine = negs.reshape(n_neg, B, S)[:, a:c].reshape(-1, S)
        losses.append(float(model.step(torch.from_numpy(seqs[a:c].copy()), torch.from_numpy(mine.copy()), loss)))
    return gather_state(st, plan, STEP['I']), losses


@pytest.mark.parametrize('world,net,loss,n_neg', STEP_CASES)
def test_sharded_seq_step_matches_single_process(world, net, loss, n_neg):
    """LSTMNet, MixtureLSTMNet (M = 2) and adaptive hinge: the sharded steps (each rank a
    contiguous slice of every minibatch, its negatives rows q*B + b of the minibatch's block,
    replicated LSTM / projection weights all-reduced) reproduce the whole-minibatch oracle."""
    res = sc.run_world(_step_job, world, (net, loss, n_neg))
    got, losses = res[0]
    params = make_params(STEP['seed'], STEP['I'], STEP['D'], net)
    batches = make_batches(STEP['seed'] + 2, STEP['I'], STEP['B'], STEP['S'], STEP['steps'], n_neg)
    ref, ref_losses = oracle_trajectory(params, batches, loss, 0.05, n_neg)
    assert_close(np.array(losses), np.array(ref_losses), 1e-5, what='losses')
    assert len(got) == len(ref)
    for k, (a, b) in enumerate(zip(got, ref)):
        assert_close(a, b.reshape(a.shape), 3e-5, what='param%d' % k)
    for r in range(1, world):
        assert res[r][1] == losses                          # every rank returns the global loss
    assert not got[0][0].any() and not got[1][0].any()      # padding row stays zero


# ------------------------------------------------------------------ ShardedImplicitSequenceModel.fit

FIT = dict(seed=17, I=37, D=8, S=6, n=47, B=9, n_iter=2)      # last minibatch: 2 rows
FIT_CASES = [(2, 'pooling', 'adaptive_hinge'), (3, 'lstm', 'pointwise'), (2, 'mixture', 'bpr'),
             (3, 'cnn', 'pointwise')]


def _fit_data():
    rs = np.random.RandomState(FIT['seed'] + 5)
    seqs = rs.randint(1, FIT['I'], (FIT['n'], FIT['S'])).astype(np.int64)
    for b in range(FIT['n']):
        seqs[b, :rs.randint(0, FIT['S'])] = 0
    return seqs


def _fit_job(rank, world, dev, rep, loss):
    from spotlight_b200.interactions import SequenceInteractions
    from spotlight_b200.sharded import ShardedImplicitSequenceModel
    rs = np.random.RandomState(FIT['seed'])
    model = ShardedImplicitSequenceModel(FIT['I'], rank, world, dev, loss=loss, representation=rep,
                                         embedding_dim=FIT['D'], n_iter=FIT['n_iter'], batch_size=FIT['B'],
                                         learning_rate=0.05, random_state=rs, num_negative_samples=3,
                                         backend=SeqBackend())
    model.fit(SequenceInteractions(_fit_data(), num_items=FIT['I']))
    net = model.gathered_net()
    params = [p.detach().numpy().copy() for p in net.parameters()]
    return params, model.epoch_losses, rs.get_state()


def _reference_fit(rep, loss, n_neg, store=None):
    """The single-process fit: the constructor's draw and set_seed, the net built as _initialize
    builds it, per epoch one cumulative shuffle and one (n_seq * n_neg, S) draw, minibatches of
    B rows, each stepped whole through the float64 oracle with dense Adagrad (parameters and
    states rounded to ``store`` after every step when given)."""
    from spotlight_b200.sequence.representations import CNNNet, LSTMNet, MixtureLSTMNet, PoolNet
    from spotlight_b200.torch_utils import set_seed
    rs = np.random.RandomState(FIT['seed'])
    set_seed(rs.randint(-10 ** 8, 10 ** 8))
    net = {'pooling': PoolNet, 'cnn': CNNNet, 'lstm': LSTMNet, 'mixture': MixtureLSTMNet}[rep](FIT['I'], FIT['D'])
    P = [p.detach().numpy().astype(np.float64).copy() for p in net.parameters()]
    names = [nm for nm, _ in net.named_parameters()]
    St = [np.zeros_like(p) for p in P]
    by = dict(zip(names, range(len(P))))
    seqs = _fit_data()
    n, S, B = FIT['n'], FIT['S'], FIT['B']
    epoch_losses = []
    for _ in range(FIT['n_iter']):
        order = np.arange(n)
        rs.shuffle(order)
        seqs = seqs[order]
        negatives = rs.randint(0, FIT['I'], (n * n_neg, S), dtype=np.int64)
        losses = []
        for lo in range(0, n, B):
            m = min(B, n - lo)
            E, bias = P[by['item_embeddings.weight']], P[by['item_biases.weight']]
            lstm = mix = convs = cnn = None
            if 'lstm.weight_ih_l0' in by:
                lstm = {k: P[by['lstm.%s_l0' % ({'w_ih': 'weight_ih', 'w_hh': 'weight_hh', 'b_ih': 'bias_ih',
                                                  'b_hh': 'bias_hh'}[k])]] for k in LSTM_KEYS}
            if 'projection.weight' in by:
                mix = dict(w=P[by['projection.weight']], b=P[by['projection.bias']], num_mixtures=net.num_mixtures)
            if rep == 'cnn':
                cnn = dict(kernel_width=list(net.kernel_width), dilation=list(net.dilation),
                           nonlinearity='tanh', residual=True)
                convs = [(P[by['cnn_%d.weight' % i]], P[by['cnn_%d.bias' % i]]) for i in range(len(net.cnn_layers))]
            r, grads = oracle_seq_step(E, bias, lstm, mix, seqs[lo:lo + m], negatives[lo * n_neg:(lo + m) * n_neg],
                                       loss, n_neg, convs, cnn)
            losses.append(float(r['loss']))
            g = {'item_embeddings.weight': r['dE'], 'item_biases.weight': r['dbias']}
            if cnn is not None:
                for i in range(len(net.cnn_layers)):
                    g['cnn_%d.weight' % i], g['cnn_%d.bias' % i] = grads[2 * i], grads[2 * i + 1]
            if lstm is not None:
                for k, nm in zip(LSTM_KEYS, ('weight_ih', 'weight_hh', 'bias_ih', 'bias_hh')):
                    g['lstm.%s_l0' % nm] = r['dlstm'][k]
            if mix is not None:
                g['projection.weight'], g['projection.bias'] = r['dmix']['w'], r['dmix']['b']
            adagrad(P, St, [g[nm] for nm in names], 0.05, store=store)
        epoch_losses.append(float(np.mean(losses)))
    return P, epoch_losses, rs


@pytest.mark.parametrize('world,rep,loss', FIT_CASES)
def test_sharded_sequence_fit_is_the_single_process_fit(world, rep, loss):
    """fit() on N ranks over two epochs: 47 sequences in minibatches of 9 (the last one has 2 rows,
    fewer than the world at 3 ranks, so a rank steps with no rows) reproduce the single-process
    replay: epoch losses, item table, bias and replicated parameters, and every rank's final
    RandomState."""
    n_neg = 3 if loss == 'adaptive_hinge' else 1
    res = sc.run_world(_fit_job, world, (rep, loss))
    # float32 parameter storage, as the model keeps: the hinge's kink and its argmax over negatives
    # turn the 1e-8 gap between float64 and float32 storage into different active terms within an
    # epoch, so a float64-stored replay is a different (equally valid) trajectory
    ref, ref_losses, rs = _reference_fit(rep, loss, n_neg, np.float32)
    want = rs.get_state()
    for r in range(world):
        got, losses, state = res[r]
        assert_close(np.array(losses), np.array(ref_losses), 1e-5, what='epoch losses')
        assert len(got) == len(ref)
        for k, (a, b) in enumerate(zip(got, ref)):
            assert_close(a, b.reshape(a.shape), 5e-5, what='param%d' % k)
        assert np.array_equal(state[1], want[1]) and state[2] == want[2]      # stream position on every rank


def test_sharded_sequence_model_rejects_unsupported_nets():
    from spotlight_b200.layers import BloomEmbedding
    from spotlight_b200.sequence.representations import PoolNet
    from spotlight_b200.sharded import ShardedImplicitSequenceModel
    with pytest.raises(ValueError):
        ShardedImplicitSequenceModel(20, 0, 1, 'cpu', embedding_dim=6, backend=SeqBackend())     # D % 4 != 0
    bloom = PoolNet(20, 8, item_embedding_layer=BloomEmbedding(20, 8, padding_idx=0))
    with pytest.raises(ValueError):
        ShardedImplicitSequenceModel(20, 0, 1, 'cpu', representation=bloom, embedding_dim=8, backend=SeqBackend())
    with pytest.raises(ValueError):
        ShardedImplicitSequenceModel(20, 0, 1, 'cpu', representation=torch.nn.Linear(2, 2), backend=SeqBackend())


# ------------------------------------------------------------------ owner update semantics

def owner_update_reference(ids, g_rows, g_bias, W, S, b, sb, lr, eps=1e-10):
    """The owner-side update in float64: every distinct id in [0, rows) sums its contributions in
    position (= peer rank) order and takes one torch.optim.Adagrad step on its row and bias; ids
    outside [0, rows) are padding slots; no other row changes.  Returns new (W, S, b, sb)."""
    W, S, b, sb = (x.astype(np.float64).copy() for x in (W, S, b, sb))
    rows = W.shape[0]
    for r in np.unique(ids):
        if r < 0 or r >= rows:
            continue
        pos = np.nonzero(ids == r)[0]            # ascending positions: rank order
        g = np.zeros(W.shape[1])
        gb = 0.0
        for p in pos:
            g += g_rows[p]
            gb += g_bias[p]
        S[r] += g * g
        W[r] -= lr * g / (np.sqrt(S[r]) + eps)
        sb[r] += gb * gb
        b[r] -= lr * gb / (np.sqrt(sb[r]) + eps)
    return W, S, b, sb


def owner_case(seed, rows, D, peers=(9, 0, 14, 5), padding=0):
    """Request lists of several peers (each ascending and distinct, one of them empty) concatenated
    in rank order, so rows repeat across peers; ``padding`` -1 slots at the end of each list."""
    rs = np.random.RandomState(seed)
    lists = []
    for k in peers:
        ids = np.sort(rs.choice(rows, size=min(k, rows), replace=False))
        lists.append(np.concatenate([ids, -np.ones(padding if k else 0, dtype=np.int64)]))
    ids = np.concatenate(lists).astype(np.int64)
    g_rows = rs.randn(len(ids), D).astype(np.float32)
    g_bias = rs.randn(len(ids)).astype(np.float32)
    g_rows[ids < 0] = 0
    g_bias[ids < 0] = 0
    W = rs.randn(rows, D).astype(np.float32)
    S = np.abs(rs.randn(rows, D)).astype(np.float32)
    b = rs.randn(rows).astype(np.float32)
    sb = np.abs(rs.randn(rows)).astype(np.float32)
    return ids, g_rows, g_bias, W, S, b, sb


def test_owner_update_reference_is_dense_adagrad_on_the_touched_rows():
    """The row-wise owner update equals the dense segmented sum + dense Adagrad the owner used to
    run (sharded_common.NumpyBackend.owner_update) with duplicate ids across peers and an empty
    peer, and leaves untouched rows and their states bit for bit."""
    import types
    ids, g_rows, g_bias, W, S, b, sb = owner_case(3, 23, 5)
    assert len(np.unique(ids)) < len(ids)                     # rows repeat across peers
    W2, S2, b2, sb2 = owner_update_reference(ids, g_rows, g_bias, W, S, b, sb, 0.05)
    st = types.SimpleNamespace(Wi=torch.from_numpy(W.copy()), sWi=torch.from_numpy(S.copy()),
                               bi=torch.from_numpy(b.copy()), sbi=torch.from_numpy(sb.copy()), lr=0.05, eps=1e-10)
    sc.NumpyBackend().owner_update(st, torch.from_numpy(ids), torch.from_numpy(g_rows), torch.from_numpy(g_bias))
    for got, want in ((st.Wi, W2), (st.sWi, S2), (st.bi, b2), (st.sbi, sb2)):
        assert_close(got.numpy(), want, 1e-6)
    untouched = np.setdiff1d(np.arange(23), ids)
    assert len(untouched) > 0
    assert np.array_equal(W2[untouched], W[untouched]) and np.array_equal(S2[untouched], S[untouched])
    assert np.array_equal(b2[untouched], b[untouched]) and np.array_equal(sb2[untouched], sb[untouched])
    # padding slots add nothing
    pids, pg, pgb, _, _, _, _ = owner_case(3, 23, 5, padding=3)
    Wp = owner_update_reference(pids, pg, pgb, W, S, b, sb, 0.05)
    keep = pids >= 0
    Wk = owner_update_reference(pids[keep], pg[keep], pgb[keep], W, S, b, sb, 0.05)
    for x, y in zip(Wp, Wk):
        assert np.array_equal(x, y)


# ------------------------------------------------------------------ resource usage

def test_owner_update_kernel_does_not_spill():
    """Every instantiation of rows_adagrad_kernel (lanes per row 1 .. 32, float4 and scalar rows)
    has no stack frame and no local memory in the built library."""
    from test_mf_resource_usage_cpu import _find, _usage
    usage = _usage()
    for lpr in (1, 2, 4, 8, 16, 32):
        for vec in (0, 1):
            r = _find(usage, 'rows_adagrad_kernelILi%dELb%dEE' % (lpr, vec))
            assert r['STACK'] == 0 and r['LOCAL'] == 0, 'rows_adagrad_kernel<%d,%d> spills: %s' % (lpr, vec, r)
