"""Generate the sequence-model default-Adam fit fixtures from the LIVE reference (build container only).

Run:  SPOTLIGHT_REFERENCE=<reference checkout> PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_seq_adam.py

A standalone companion of make_golden.py (whose helpers it uses): it writes only the
``fit_<net>_adam`` fixtures, so the existing fixtures are not regenerated.  Each records two epochs
of the reference's ``ImplicitSequenceModel.fit`` with its default optimizer,
``optim.Adam(params, weight_decay=l2, lr=learning_rate)`` (spotlight/sequence/implicit.py), set
through ``learning_rate`` and ``l2``: the initial and final state_dict, the sequences, the epoch
losses, the RandomState afterwards and ``predict`` of one sequence.  500 items and 16 sequences of
length 6 a minibatch: a minibatch references well under half the rows, so most rows miss several
Adam steps between touches (and, with ``l2 > 0``, are still moved by the weight decay).
"""

import contextlib
import io
import os
import sys

import numpy as np

sys.dont_write_bytecode = True
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import make_golden as mg  # noqa: E402
import torch  # noqa: E402

from spotlight.interactions import SequenceInteractions  # noqa: E402
from spotlight.sequence.implicit import ImplicitSequenceModel  # noqa: E402


def seq_adam_fit_case(name, loss, representation, l2, num_items=500, dim=8, n_seq=64, S=6, batch=16,
                      n_iter=2, lr=1e-2, seed=5):
    rs = np.random.RandomState(seed)
    seqs = rs.randint(1, num_items, (n_seq, S)).astype(np.int32)
    for b in range(0, n_seq, 2):
        seqs[b, :rs.randint(0, S)] = 0
    inter = SequenceInteractions(seqs, num_items=num_items)
    model = ImplicitSequenceModel(loss=loss, representation=representation, embedding_dim=dim,
                                  batch_size=batch, n_iter=n_iter, l2=l2, learning_rate=lr,
                                  random_state=np.random.RandomState(seed))
    model._initialize(inter)
    assert type(model._optimizer) is torch.optim.Adam
    out = {('init.' + k): mg._np(v) for k, v in model._net.state_dict().items()}
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        model.fit(inter, verbose=True)
    losses = [float(line.split('loss')[1]) for line in buf.getvalue().strip().split('\n')]
    out.update({('final.' + k): mg._np(v) for k, v in model._net.state_dict().items()})
    out.update(mg._rs_state(model._random_state))
    out.update(seqs=seqs, epoch_losses=np.array(losses), num_items=np.int64(num_items), dim=np.int64(dim),
               batch=np.int64(batch), n_iter=np.int64(n_iter), seed=np.int64(seed), lr=np.float64(lr),
               l2=np.float64(l2), loss=np.array(loss), representation=np.array(representation),
               predict=model.predict(seqs[1]))
    np.savez_compressed(os.path.join(mg.HERE, name + '.npz'), **out)
    print(name, 'epoch losses', losses)


if __name__ == '__main__':
    seq_adam_fit_case('fit_pool_adam', 'bpr', 'pooling', l2=0.0)
    seq_adam_fit_case('fit_cnn_adam', 'pointwise', 'cnn', l2=1e-3)
    seq_adam_fit_case('fit_lstm_adam', 'bpr', 'lstm', l2=1e-2)
