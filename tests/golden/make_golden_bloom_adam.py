"""Generate the hashed-table default-Adam fit fixtures from the LIVE reference (build container only).

Run:  SPOTLIGHT_REFERENCE=<reference checkout> PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_bloom_adam.py

Two fits of two epochs of the reference's ``ImplicitFactorizationModel.fit`` with its default
optimizer, ``torch.optim.Adam(weight_decay=l2, lr=learning_rate)``, on a ``BilinearNet`` with
``BloomEmbedding`` layers (padding id 0):

* ``fit_bloom_adam_bpr.npz``: Bloom item layer (H = 3), plain user table, bpr, l2 = 0;
* ``fit_bloom_adam_both.npz``: Bloom user (H = 2) and item (H = 3) layers, adaptive hinge with
  3 negatives, l2 = 1e-3.

The tables are large against the minibatch (64 interactions, a few hundred hashed rows out of
400-1000), so rows miss several steps between touches.  Each fixture records the initial and final
``state_dict``, the interactions, the epoch losses, the RandomState key and position after the
constructor and after fit, and ``predict`` for one user.
"""

import contextlib
import io
import os
import sys

import numpy as np

sys.dont_write_bytecode = True
sys.path.insert(0, os.environ['SPOTLIGHT_REFERENCE'])

import torch  # noqa: E402

from spotlight.factorization.implicit import ImplicitFactorizationModel  # noqa: E402
from spotlight.factorization.representations import BilinearNet  # noqa: E402
from spotlight.interactions import Interactions  # noqa: E402
from spotlight.layers import BloomEmbedding, ScaledEmbedding  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
torch.set_num_threads(1)

FITS = [
    # name, loss, Hu (0 = plain), Hi, l2, n_neg
    ('fit_bloom_adam_bpr', 'bpr', 0, 3, 0.0, 5),
    ('fit_bloom_adam_both', 'adaptive_hinge', 2, 3, 1e-3, 3),
]


def fit(name, loss, Hu, Hi, l2, n_neg):
    U, I, D, ratio_u, ratio_i, n, B, lr = 800, 2000, 8, 0.5, 0.5, 1200, 64, 1e-2
    rs = np.random.RandomState(23)
    users = rs.randint(0, U, n).astype(np.int32)
    items = rs.randint(0, I, n).astype(np.int32)
    inter = Interactions(users, items, num_users=U, num_items=I)
    torch.manual_seed(23)
    ue = BloomEmbedding(U, D, compression_ratio=ratio_u, num_hash_functions=Hu) if Hu else ScaledEmbedding(U, D)
    ie = BloomEmbedding(I, D, compression_ratio=ratio_i, num_hash_functions=Hi)
    rep = BilinearNet(U, I, D, user_embedding_layer=ue, item_embedding_layer=ie)
    with torch.no_grad():
        rep.user_biases.weight.normal_(0, 0.1)
        rep.item_biases.weight.normal_(0, 0.1)
    model = ImplicitFactorizationModel(loss=loss, embedding_dim=D, batch_size=B, n_iter=2, l2=l2,
                                       learning_rate=lr, representation=rep, num_negative_samples=n_neg,
                                       random_state=np.random.RandomState(24))
    model._initialize(inter)
    out = {'init.' + k: v.detach().numpy().copy() for k, v in model._net.state_dict().items()}
    st = model._random_state.get_state()
    out.update(rs0_key=st[1].copy(), rs0_pos=np.int64(st[2]))
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        model.fit(inter, verbose=True)
    losses = [float(l.split('loss')[1]) for l in buf.getvalue().strip().split('\n') if l.startswith('Epoch')]
    out.update({'final.' + k: v.detach().numpy().copy() for k, v in model._net.state_dict().items()})
    st = model._random_state.get_state()
    out.update(rs_key=st[1].copy(), rs_pos=np.int64(st[2]), epoch_losses=np.array(losses),
               users=users, items=items, num_users=np.int64(U), num_items=np.int64(I), dim=np.int64(D),
               loss=np.array(loss), user_H=np.int64(Hu), item_H=np.int64(Hi), user_ratio=np.float64(ratio_u),
               item_ratio=np.float64(ratio_i), batch=np.int64(B), n_iter=np.int64(2), lr=np.float64(lr),
               l2=np.float64(l2), n_neg=np.int64(n_neg), predict_user=np.int64(3),
               predict=model.predict(3).astype(np.float32))
    np.savez_compressed(os.path.join(HERE, name + '.npz'), **out)
    print(name, losses)


if __name__ == '__main__':
    for f in FITS:
        fit(*f)
