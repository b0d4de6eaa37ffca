"""Generate the hashed-table fit fixture from the LIVE reference (build container only).

Run:  SPOTLIGHT_REFERENCE=<reference checkout> PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_bloom_fit.py

A standalone companion of make_golden.py: it writes only ``fit_bloom_adagrad.npz``, two epochs of
the reference's ``ImplicitFactorizationModel.fit`` with a ``BilinearNet`` whose item layer is a
``BloomEmbedding`` (H = 3, padding id 0), bpr, D = 16, ``torch.optim.Adagrad`` without weight
decay.  It records the initial and final ``state_dict``, the interactions, the epoch losses, the
RandomState key and position after the constructor and after fit, and ``predict`` for one user.
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


def main():
    U, I, D, H, ratio, n, B, lr = 60, 400, 16, 3, 0.3, 1500, 128, 0.05
    rs = np.random.RandomState(17)
    users = rs.randint(0, U, n).astype(np.int32)
    items = rs.randint(0, I, n).astype(np.int32)
    inter = Interactions(users, items, num_users=U, num_items=I)
    torch.manual_seed(17)
    rep = BilinearNet(U, I, D, user_embedding_layer=ScaledEmbedding(U, D),
                      item_embedding_layer=BloomEmbedding(I, D, compression_ratio=ratio, num_hash_functions=H))
    with torch.no_grad():
        rep.user_biases.weight.normal_(0, 0.1)
        rep.item_biases.weight.normal_(0, 0.1)
    model = ImplicitFactorizationModel(loss='bpr', embedding_dim=D, batch_size=B, n_iter=2, representation=rep,
                                       optimizer_func=lambda p: torch.optim.Adagrad(p, lr=lr),
                                       random_state=np.random.RandomState(18))
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
               bloom_H=np.int64(H), bloom_ratio=np.float64(ratio), batch=np.int64(B), n_iter=np.int64(2),
               lr=np.float64(lr), predict_user=np.int64(3), predict=model.predict(3).astype(np.float32))
    np.savez_compressed(os.path.join(HERE, 'fit_bloom_adagrad.npz'), **out)
    print('fit_bloom_adagrad', losses)


if __name__ == '__main__':
    main()
