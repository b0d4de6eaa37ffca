"""Generate the Bloom-item sequence golden vectors from the LIVE reference (build container only).

Run:  SPOTLIGHT_REFERENCE=<reference checkout> PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_seq_bloom.py

A standalone companion of make_golden.py (whose helpers it uses): it writes only the fixtures of
sequence nets with a ``BloomEmbedding`` item layer, so the existing fixtures are not regenerated.

* One-step fixtures (``seq_bloom_*``): the reference's CNNNet (two layers, dilation), LSTMNet and
  MixtureLSTMNet (4 tastes) over a BloomEmbedding with 1, 2 or 4 hashes on a small table where
  ids collide -- an id of the batch with two hashes on one row, ids on the frozen row 0 -- with
  the adaptive hinge among the losses.  Each records what make_golden.seq_case records: the
  state_dict, the minibatch, the negatives the reference drew, its predictions, loss, final
  representation and every parameter's ``.grad``.
* ``fit_bloom_lstm_adagrad``: two epochs of the reference's ImplicitSequenceModel with a Bloom
  LSTMNet (4 hashes, ratio 0.5) under ``torch.optim.Adagrad`` without weight decay: initial and
  final parameters, per-epoch losses, the RandomState afterwards and one ``predict``.
"""

import contextlib
import io
import os
import sys

import numpy as np

sys.dont_write_bytecode = True
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))

import make_golden as mg  # noqa: E402
import torch  # noqa: E402

from spotlight.interactions import SequenceInteractions  # noqa: E402
from spotlight.layers import BloomEmbedding  # noqa: E402
from spotlight.sequence.implicit import ImplicitSequenceModel  # noqa: E402
from spotlight.sequence.representations import CNNNet, LSTMNet, MixtureLSTMNet  # noqa: E402

from oracle.murmur import bloom_rows  # noqa: E402


def _net(kind, num_items, dim, emb):
    if kind == 'cnn':
        return CNNNet(num_items, dim, kernel_width=(3, 2), dilation=(1, 2), num_layers=2,
                      item_embedding_layer=emb)
    if kind == 'lstm':
        return LSTMNet(num_items, dim, item_embedding_layer=emb)
    return MixtureLSTMNet(num_items, dim, num_mixtures=4, item_embedding_layer=emb)


def step_case(name, kind, loss, num_items, dim, batch, S, H, ratio, n_neg=3, seed=21):
    """make_golden.seq_case for a Bloom-embedded CNNNet / LSTMNet / MixtureLSTMNet."""
    rs = np.random.RandomState(seed)
    seqs = rs.randint(1, num_items, (batch, S)).astype(np.int64)
    for b in range(batch):                     # random left zero-pad
        if b % 3 == 0:
            seqs[b, :rs.randint(0, S)] = 0
    seqs[1, :] = 0                             # one fully padded row
    M = int(ratio * num_items)
    rows = bloom_rows(np.arange(num_items), H, M)
    if H >= 2:                                 # an id with two hashes on one row
        dup = [i for i in range(1, num_items) if len(np.unique(rows[i])) < H]
        seqs[2, -1] = dup[0]
    on0 = [i for i in range(1, num_items) if (rows[i] == 0).any()]
    seqs[3, -1] = on0[0]                       # an id on the frozen row
    inter = SequenceInteractions(seqs.astype(np.int32), num_items=num_items)
    torch.manual_seed(seed)
    emb = BloomEmbedding(num_items, dim, compression_ratio=ratio, num_hash_functions=H, padding_idx=0)
    model = ImplicitSequenceModel(loss=loss, representation=_net(kind, num_items, dim, emb), embedding_dim=dim,
                                  batch_size=batch, num_negative_samples=n_neg,
                                  random_state=np.random.RandomState(seed + 1))
    model._initialize(inter)
    net = model._net
    with torch.no_grad():
        g = torch.Generator().manual_seed(seed)
        net.item_biases.weight.copy_(torch.randn(net.item_biases.weight.shape, generator=g) * 0.1)
        net.item_biases.weight[0] = 0.0
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
    out.update(seqs=seqs, negs=negs, pos=mg._np(pos), neg=mg._np(neg), final=mg._np(final),
               loss=np.float32(lv.item()), n_neg=np.int64(n_neg), num_items=np.int64(num_items),
               dim=np.int64(dim), bloom_H=np.int64(H), bloom_ratio=np.float64(ratio), net=np.str_(kind),
               loss_name=np.str_(loss))
    np.savez_compressed(os.path.join(mg.HERE, name + '.npz'), **out)
    print(name, 'loss', lv.item())


def fit_case():
    I, D, H, ratio, n_seq, S, B, lr, seed = 120, 16, 4, 0.5, 48, 8, 16, 0.05, 31
    rs = np.random.RandomState(seed)
    seqs = rs.randint(1, I, (n_seq, S)).astype(np.int32)
    for b in range(0, n_seq, 2):
        seqs[b, :rs.randint(0, S)] = 0
    inter = SequenceInteractions(seqs, num_items=I)
    torch.manual_seed(seed)
    emb = BloomEmbedding(I, D, compression_ratio=ratio, num_hash_functions=H, padding_idx=0)
    model = ImplicitSequenceModel(loss='bpr', representation=LSTMNet(I, D, item_embedding_layer=emb),
                                  embedding_dim=D, batch_size=B, n_iter=2,
                                  optimizer_func=lambda p: torch.optim.Adagrad(p, lr=lr),
                                  random_state=np.random.RandomState(seed))
    model._initialize(inter)
    out = {('init.' + k): mg._np(v) for k, v in model._net.state_dict().items()}
    st = model._random_state.get_state()
    out.update(rs0_key=st[1].copy(), rs0_pos=np.int64(st[2]))
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        model.fit(inter, verbose=True)
    losses = [float(line.split('loss')[1]) for line in buf.getvalue().strip().split('\n')]
    out.update({('final.' + k): mg._np(v) for k, v in model._net.state_dict().items()})
    out.update(mg._rs_state(model._random_state))
    out.update(seqs=seqs, epoch_losses=np.array(losses), num_items=np.int64(I), dim=np.int64(D),
               bloom_H=np.int64(H), bloom_ratio=np.float64(ratio), batch=np.int64(B), n_iter=np.int64(2),
               lr=np.float64(lr), seed=np.int64(seed), predict=model.predict(seqs[1]))
    np.savez_compressed(os.path.join(mg.HERE, 'fit_bloom_lstm_adagrad.npz'), **out)
    print('fit_bloom_lstm_adagrad', losses)


if __name__ == '__main__':
    step_case('seq_bloom_cnn_bpr', 'cnn', 'bpr', num_items=80, dim=16, batch=8, S=9, H=2, ratio=0.25)
    step_case('seq_bloom_lstm_adaptive', 'lstm', 'adaptive_hinge', num_items=80, dim=16, batch=8, S=9, H=4,
              ratio=0.2)
    step_case('seq_bloom_mixture_pointwise', 'mixture', 'pointwise', num_items=80, dim=16, batch=8, S=9, H=1,
              ratio=0.3)
    fit_case()
