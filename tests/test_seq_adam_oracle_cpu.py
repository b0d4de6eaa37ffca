"""Lazy-exact Adam for the sequence models without the GPU.

* The scheme the sequence step ships (csrc/seq.cu seq_adam_prepass_kernel / seq_reduce_adam_kernel):
  every item row and bias the minibatch references caught up through step t - 1 before the forward,
  the real step t on the rows with a gradient, a flush at the end of fit() -- in NumPy float64
  (oracle/adam.py LazyAdamTable), with dense Adam on the net's own parameters and the float64
  sequence oracles for the gradients, driven over the reference's own minibatch stream, against
  the trajectories the live reference recorded with its default dense Adam
  (tests/golden/make_golden_seq_adam.py).
* FusedAdam.step() on CPU tensors of the LSTM nets is ordinary Adam.
* The lazy-Adam kernels compile without register spills (sm_90a).
"""
import numpy as np
import pytest
import torch

from conftest import assert_close, load_golden
from oracle import lstm_cases as lc
from oracle import seq_cases as sc
from oracle.adam import LazyAdamTable
from test_mf_resource_usage_cpu import _find, _usage

LSTM_NAMES = {'w_ih': 'lstm.weight_ih_l0', 'w_hh': 'lstm.weight_hh_l0', 'b_ih': 'lstm.bias_ih_l0',
              'b_hh': 'lstm.bias_hh_l0'}


def _reference_minibatches(g):
    """The reference fit()'s stream: the constructor's seed draw, then per epoch a cumulative
    shuffle of the sequences and one negative draw per minibatch (sequence/implicit.py)."""
    I, B = int(g['num_items']), int(g['batch'])
    rs = np.random.RandomState(int(g['seed']))
    rs.randint(-10**8, 10**8)
    seqs = g['seqs'].astype(np.int64)
    epochs = []
    for _ in range(int(g['n_iter'])):
        idx = np.arange(len(seqs))
        rs.shuffle(idx)
        seqs = seqs[idx]
        epochs.append([(seqs[lo:lo + B], rs.randint(0, I, seqs[lo:lo + B].shape, dtype=np.int64))
                       for lo in range(0, len(seqs), B)])
    return epochs, rs


def _oracle_step(net, loss, tabs, seqs, negs):
    """float64 gradients of every parameter, keyed by state_dict name."""
    E, bias = tabs['item_embeddings.weight'].w, tabs['item_biases.weight'].w
    if net == 'lstm':
        lstm = {k: tabs[n].w for k, n in LSTM_NAMES.items()}
        r = lc.oracle_step(dict(E=E, bias=bias, lstm=lstm, seqs=seqs, negs=negs, loss=loss, n_neg=1))
        grads = {n: r['dlstm'][k] for k, n in LSTM_NAMES.items()}
    elif net == 'cnn':
        convs = [(tabs['cnn_0.weight'].w, tabs['cnn_0.bias'].w)]
        case = dict(E=E, bias=bias, seqs=seqs, negs=negs, loss=loss, n_neg=1, convs=convs,
                    cnn=dict(kernel_width=[3], dilation=[1], nonlinearity='tanh', residual=True))
        r = sc.oracle_step(case)
        grads = {'cnn_0.weight': r['dconvs'][0][0], 'cnn_0.bias': r['dconvs'][0][1]}
    else:
        r = sc.oracle_step(dict(E=E, bias=bias, seqs=seqs, negs=negs, loss=loss, n_neg=1, cnn=None))
        grads = {}
    grads['item_embeddings.weight'], grads['item_biases.weight'] = r['dE'], r['dbias']
    return float(r['loss']), grads


FITS = [('fit_pool_adam', 'pooling'), ('fit_cnn_adam', 'cnn'), ('fit_lstm_adam', 'lstm')]


@pytest.mark.parametrize('name,net', FITS, ids=[f[0] for f in FITS])
def test_lazy_scheme_reproduces_reference_default_adam_fit(name, net):
    """Epoch losses at 1e-5, final parameters at 2e-3 of their scale (Adam's m / sqrt(v) turns
    last-bit gradient differences on near-zero components into fractions of a step, as in
    test_oracle_port.test_lazy_adam_scheme_reproduces_reference_default_adam_fit), RandomState
    position exact.  The item table and bias are lazy: a row is caught up only when a minibatch
    references it (padding id included) and at the final flush."""
    g = load_golden(name)
    loss = str(g['loss'])
    lr, l2 = float(g['lr']), float(g['l2'])
    lazy = ('item_embeddings.weight', 'item_biases.weight')
    tabs = {k[5:]: LazyAdamTable(v, lr=lr, weight_decay=l2) for k, v in g.items() if k.startswith('init.')}
    epochs, rs = _reference_minibatches(g)
    t, losses, missed = 0, [], 0
    for batches in epochs:
        ep = []
        for seqs, negs in batches:
            t += 1
            ref_rows = np.concatenate([seqs.ravel(), negs.ravel()])
            for k in lazy:
                tabs[k].catch_up(ref_rows, t - 1)            # before the forward sees the weights
            lval, grads = _oracle_step(net, loss, tabs, seqs, negs)
            ep.append(lval)
            for k, tab in tabs.items():
                gr = np.asarray(grads[k], dtype=np.float64).reshape(tab.w.shape)
                if k in lazy:                                # rows with an all-zero gradient are not touched
                    rows = np.flatnonzero(np.abs(gr.reshape(gr.shape[0], -1)).sum(axis=1) > 0)
                    missed += int((tab.last[1:] < t - 1).sum())
                else:                                        # the net's own parameters: dense Adam
                    rows = np.arange(tab.w.shape[0])
                tab.apply(rows, gr[rows], t)
        losses.append(float(np.mean(ep)))
    for tab in tabs.values():
        tab.flush(t)
    assert missed > 0, 'no row missed a step: the case does not exercise the catch-up'
    assert_close(np.array(losses), g['epoch_losses'], 1e-5, what='epoch losses')
    for k, tab in tabs.items():
        assert_close(tab.w, g['final.' + k], 2e-3, atol=1e-7, what=k)
    st = rs.get_state()
    assert (st[1] == g['rs_key']).all() and st[2] == int(g['rs_pos'])


@pytest.mark.parametrize('net', ['lstm', 'mixture'])
def test_fused_adam_step_equals_torch_adam(net):
    """FusedAdam.step() on CPU tensors of an LSTMNet / MixtureLSTMNet (LSTM weights of (4D, D), a
    mixture projection) is ordinary Adam on every parameter: none of them is a lazily updated
    table, so flush() pairs nothing."""
    from spotlight_b200.optim import FusedAdam
    from spotlight_b200.sequence.representations import LSTMNet, MixtureLSTMNet
    torch.manual_seed(0)
    make = (lambda: LSTMNet(50, 8)) if net == 'lstm' else (lambda: MixtureLSTMNet(50, 8, num_mixtures=2))
    a, b = make(), make()
    b.load_state_dict(a.state_dict())
    mine = FusedAdam(a.parameters(), lr=1e-2, weight_decay=1e-3)
    ref = torch.optim.Adam(b.parameters(), lr=1e-2, weight_decay=1e-3)
    for _ in range(4):
        for p, q in zip(a.parameters(), b.parameters()):
            g = torch.randn_like(p)
            p.grad, q.grad = g.clone(), g.clone()
        mine.step()
        ref.step()
    assert mine.steps_taken == 4
    for (k, x), (_, y) in zip(a.state_dict().items(), b.state_dict().items()):
        assert torch.allclose(x, y, rtol=1e-5, atol=1e-7), k


def test_fused_adam_rejects_sparse_gradients():
    """A sparse embedding (sparse=True) hands the optimizer a sparse gradient: FusedAdam refuses it
    with a clear error, as torch.optim.Adam does."""
    from spotlight_b200.optim import FusedAdam
    emb = torch.nn.Embedding(10, 4, sparse=True)
    emb(torch.tensor([1, 2])).sum().backward()
    with pytest.raises(RuntimeError, match='sparse'):
        FusedAdam(emb.parameters()).step()
    with pytest.raises(RuntimeError):
        torch.optim.Adam(emb.parameters()).step()


LPRS = (1, 2, 4, 8, 16, 32)
CASES = [('%s<%d,%s>' % (k, l, h), '%sILi%dELb%dEE' % (k, l, int(h == 'true')))
         for k in ('seq_adam_prepass_kernel', 'seq_reduce_adam_kernel') for l in LPRS for h in ('false', 'true')] + \
        [('adam_flush_table_kernel<%d>' % l, 'adam_flush_table_kernelILi%dEE' % l) for l in LPRS]


@pytest.mark.parametrize('name,mangled', CASES, ids=[c[0] for c in CASES])
def test_lazy_adam_kernels_do_not_spill(name, mangled):
    r = _find(_usage(), mangled)
    assert r['STACK'] == 0 and r['LOCAL'] == 0, '%s spills: %s' % (name, r)
