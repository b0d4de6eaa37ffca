"""Generate the MixtureLSTMNet golden vectors from the LIVE reference (build container only).

Run:  SPOTLIGHT_REFERENCE=<reference checkout> PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_mixture.py

A standalone companion of make_golden_lstm.py (whose helpers, and make_golden.py's, it uses): it
writes only the four MixtureLSTMNet fixtures.  Each step fixture records the state_dict, the
minibatch and the negatives the reference drew, its predictions, loss, representations and every
parameter's ``.grad`` for the reference's ``MixtureLSTMNet``.  The compact D = 128 fixture stores
seeds instead of the LSTM and projection weight matrices and their gradients at seeded rows
(``oracle.lstm_cases.seeded_lstm_weights`` / ``sampled_grad_rows``,
``oracle.mixture_cases.seeded_projection_weight`` / ``sampled_proj_rows``).
"""

import os
import sys

import numpy as np

sys.dont_write_bytecode = True
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))

import make_golden as mg  # noqa: E402
import torch  # noqa: E402

from spotlight.interactions import SequenceInteractions  # noqa: E402
from spotlight.sequence.implicit import ImplicitSequenceModel  # noqa: E402
from spotlight.sequence.representations import MixtureLSTMNet  # noqa: E402

from oracle import lstm_cases, mixture_cases  # noqa: E402


def mixture_step_case(name, loss, num_items, dim, batch, S, M=4, n_neg=3, seed=11, compact=False):
    """make_golden_lstm.lstm_step_case for the reference's MixtureLSTMNet."""
    rs = np.random.RandomState(seed)
    seqs = rs.randint(1, num_items, (batch, S)).astype(np.int64)
    for b in range(batch):                     # random left zero-pad
        pad = rs.randint(0, S)
        if b % 3 == 0:
            seqs[b, :pad] = 0
    seqs[1, :] = 0                             # one fully padded row
    seqs[2, -1] = num_items - 1
    inter = SequenceInteractions(seqs.astype(np.int32), num_items=num_items)
    torch.manual_seed(seed)
    rep = MixtureLSTMNet(num_items, dim, num_mixtures=M)
    model = ImplicitSequenceModel(loss=loss, representation=rep, embedding_dim=dim,
                                  batch_size=batch, num_negative_samples=n_neg,
                                  random_state=np.random.RandomState(seed + 1))
    model._initialize(inter)
    net = model._net
    with torch.no_grad():
        g = torch.Generator().manual_seed(seed)
        net.item_biases.weight.copy_(torch.randn(net.item_biases.weight.shape, generator=g) * 0.1)
        net.item_biases.weight[0] = 0.0
        # the projection weight at 4x nn.Conv1d's init widens the mixture logits; at these item
        # embedding scales the weights stay near uniform all the same, and the oracle's own cases
        # (oracle.mixture_cases) are the ones that measure the softmax path
        if compact:
            w_ih, w_hh = lstm_cases.seeded_lstm_weights(seed + 100, dim)
            net.lstm.weight_ih_l0.copy_(torch.from_numpy(w_ih))
            net.lstm.weight_hh_l0.copy_(torch.from_numpy(w_hh))
            net.projection.weight.copy_(torch.from_numpy(mixture_cases.seeded_projection_weight(seed + 100, dim, M)))
        net.projection.weight.mul_(4.0)
    out = dict(mg._state(net))
    out.update(mg._rs_state(model._random_state))
    rs_copy = np.random.RandomState()
    rs_copy.set_state(model._random_state.get_state())
    sv = torch.from_numpy(seqs)
    # replay of spotlight/sequence/implicit.py:230-253
    user_rep, final = net.user_representation(sv)
    pos = net(user_rep, sv)
    if loss == 'adaptive_hinge':
        neg = model._get_multiple_negative_predictions(sv.size(), user_rep, n=n_neg)
        negs = rs_copy.randint(0, num_items, (n_neg * batch, S), dtype=np.int64)
    else:
        neg = model._get_negative_prediction(sv.size(), user_rep)
        negs = rs_copy.randint(0, num_items, (batch, S), dtype=np.int64)
    assert rs_copy.get_state()[2] == model._random_state.get_state()[2]
    model._optimizer.zero_grad()
    lv = model._loss_func(pos, neg, mask=(sv != 0))
    lv.backward()
    out.update(mg._grads(net))
    if compact:
        rows = lstm_cases.sampled_grad_rows(seed + 100, dim)
        for k in ('weight_ih_l0', 'weight_hh_l0'):
            assert np.array_equal(out.pop('sd.lstm.' + k), getattr(net.lstm, k).detach().numpy())
            out['grad.lstm.' + k] = out['grad.lstm.' + k][rows]
        prows = mixture_cases.sampled_proj_rows(seed + 100, dim, M)
        w = out.pop('sd.projection.weight')
        assert np.array_equal(w, mixture_cases.seeded_projection_weight(seed + 100, dim, M) * np.float32(4.0))
        out['grad.projection.weight'] = out['grad.projection.weight'][prows]
        out.update(lstm_weight_seed=np.int64(seed + 100), grad_rows=rows, proj_weight_seed=np.int64(seed + 100),
                   proj_weight_scale=np.float32(4.0), proj_rows=prows)
    out.update(seqs=seqs, negs=negs, pos=mg._np(pos), neg=mg._np(neg), final=mg._np(final),
               loss=np.float32(lv.item()), n_neg=np.int64(n_neg), num_items=np.int64(num_items),
               dim=np.int64(dim), num_mixtures=np.int64(M))
    if not compact:
        out['user_rep'] = mg._np(user_rep)
    np.savez_compressed(os.path.join(mg.HERE, name + '.npz'), **out)
    print(name, 'loss', lv.item())


if __name__ == '__main__':
    mixture_step_case('mixture_pointwise', 'pointwise', num_items=61, dim=16, batch=10, S=9)
    mixture_step_case('mixture_adaptive_hinge', 'adaptive_hinge', num_items=61, dim=16, batch=8, S=11)
    # D = 128: the wgmma projections and a 4-CTA cluster recurrence
    mixture_step_case('mixture_bpr_d128', 'bpr', num_items=61, dim=128, batch=10, S=25, compact=True)
    mg.seq_fit_case('fit_mixture_sgd', 'bpr', 'mixture', 40, 8, 50, 6, 16, 2)
