"""Explicit-feedback factorization model with the reference's estimator API
(spotlight/factorization/explicit.py:22-284): same constructor arguments,
``fit(interactions, verbose)``, ``predict(user_ids, item_ids=None)``, private
attributes (``_net``, ``_optimizer``, ``_random_state``, ``_num_users``,
``_num_items``) and error behaviour.

Losses (spotlight/losses.py:169-244), on the score ``s`` of each rated pair:
``regression`` ``(r - s)^2``; ``poisson`` ``exp(s) - r log exp(s)`` (fit applies
``exp`` before the loss); ``logistic`` BCE with logits against ``clamp(r, 0, 1)``.
There are no negatives: each epoch consumes the ``RandomState`` only through one
``shuffle`` of ``arange(n)``, exactly as the reference does.

Four routes, chosen per model, as in :mod:`spotlight_b200.factorization.implicit`:

``epoch pipeline``   BilinearNet with plain tables + a fused optimizer (including the
                     default :class:`~spotlight_b200.optim.FusedAdam`): the whole epoch is
                     enqueued by one C call, one gradient term per interaction, and the
                     host reads the per-batch losses once at the end.  Fused SGD / Adagrad
                     at D in {8, 16, 32, 64, 128} run the planned two-kernel step (its plan
                     one step ahead on a side stream); lazy Adam and other D the
                     first-generation kernels.
``fused autograd``   BilinearNet with plain tables + any ``torch.optim`` optimizer: one
                     fused op per minibatch fills dense ``.grad``.
``bloom``            BilinearNet with ``BloomEmbedding`` user and / or item layers + fused SGD /
                     Adagrad: one fused hashed-table step per minibatch updates the rows it
                     touches in place (no dense gradient); the host reads the per-batch
                     losses once per epoch.  As on the other fused routes, weight decay
                     applies to the touched rows only.
``generic``          custom ``representation``, sparse models, and Bloom layers under any
                     other optimizer: the reference's loop over ``net(...)`` and this
                     package's rating losses.

Ratings go to the device once per ``fit()`` as float32.  A float64 rating array is
therefore trained in float32 (the reference promotes the loss to float64); integer-valued
ratings give the same result either way.
"""

import ctypes

import numpy as np
import torch
import torch.optim as optim

from spotlight_b200 import _lib, ops
from spotlight_b200.factorization import implicit
from spotlight_b200.factorization._components import _predict_process_ids
from spotlight_b200.factorization.implicit import (_NO_CPU, DEVICE_SHUFFLE_MIN, _fused_optimizer, _plan_stream,
                                                   _side_stream, _to_device_narrow)
from spotlight_b200.factorization.representations import BilinearNet
from spotlight_b200.helpers import _repr_model
from spotlight_b200.losses import logistic_loss, poisson_loss, regression_loss
from spotlight_b200.rng import (SHUFFLE_DEVICE_MAX, permute_ids, shuffle_begin, shuffle_end,
                                shuffled_order_device)
from spotlight_b200.torch_utils import cpu, gpu, minibatch, set_seed, shuffled_order


class ExplicitFactorizationModel(object):
    """Explicit feedback matrix factorization (ratings).

    Parameters (identical to the reference, explicit.py:68-79)
    ----------
    loss: 'regression' | 'poisson' | 'logistic'
    embedding_dim, n_iter, batch_size, l2, learning_rate
    optimizer_func: callable(params) -> torch optimizer; default is the reference's dense
        ``Adam(weight_decay=l2, lr=learning_rate)``, run as the row-wise lazy-exact
        :class:`~spotlight_b200.optim.FusedAdam` on plain tables.
    use_cuda: must be True to ``fit`` / ``predict``.
    representation: optional custom network module.
    sparse: use sparse gradients for embedding layers.
    random_state: ``numpy.random.RandomState`` driving the epoch shuffles.
    """

    def __init__(self, loss='regression', embedding_dim=32, n_iter=10, batch_size=256, l2=0.0,
                 learning_rate=1e-2, optimizer_func=None, use_cuda=False, representation=None,
                 sparse=False, random_state=None):

        assert loss in ('regression', 'poisson', 'logistic')

        self._loss = loss
        self._embedding_dim = embedding_dim
        self._n_iter = n_iter
        self._learning_rate = learning_rate
        self._batch_size = batch_size
        self._l2 = l2
        self._use_cuda = use_cuda
        self._representation = representation
        self._sparse = sparse
        self._optimizer_func = optimizer_func
        self._random_state = random_state or np.random.RandomState()

        self._num_users = None
        self._num_items = None
        self._net = None
        self._optimizer = None
        self._loss_func = None

        # same stream position as the reference (explicit.py:103-104)
        set_seed(self._random_state.randint(-10**8, 10**8), cuda=self._use_cuda)

    def __repr__(self):
        return _repr_model(self)

    @property
    def _initialized(self):
        return self._net is not None

    def _initialize(self, interactions):
        if not self._use_cuda:
            raise RuntimeError(_NO_CPU)
        (self._num_users, self._num_items) = (interactions.num_users, interactions.num_items)

        if self._representation is not None:
            self._net = gpu(self._representation, self._use_cuda)
        else:
            self._net = gpu(BilinearNet(self._num_users, self._num_items, self._embedding_dim,
                                        sparse=self._sparse), self._use_cuda)

        if self._optimizer_func is None:
            if isinstance(self._net, BilinearNet) and self._net.plain_tables() and not self._sparse:
                # optim.Adam(weight_decay=l2, lr) (explicit.py:132-137) as the row-wise
                # lazy-exact Adam: same trajectory, O(batch) instead of O(table) per step
                from spotlight_b200.optim import FusedAdam
                self._optimizer = FusedAdam(self._net.parameters(), weight_decay=self._l2,
                                            lr=self._learning_rate)
            else:
                self._optimizer = optim.Adam(self._net.parameters(), weight_decay=self._l2,
                                             lr=self._learning_rate)
        else:
            self._optimizer = self._optimizer_func(self._net.parameters())

        self._loss_func = {'regression': regression_loss, 'poisson': poisson_loss,
                           'logistic': logistic_loss}[self._loss]

    def _check_input(self, user_ids, item_ids, allow_items_none=False):
        user_id_max = user_ids if isinstance(user_ids, int) else user_ids.max()
        if user_id_max >= self._num_users:
            raise ValueError('Maximum user id greater than number of users in model.')
        if allow_items_none and item_ids is None:
            return
        item_id_max = item_ids if isinstance(item_ids, int) else item_ids.max()
        if item_id_max >= self._num_items:
            raise ValueError('Maximum item id greater than number of items in model.')

    def _route(self):
        net = self._net
        fused_kind = getattr(self._optimizer, 'fused_kind', None)
        fusable = isinstance(net, BilinearNet) and net.plain_tables()
        if fusable and fused_kind is not None:
            return 'epoch'
        if fusable and not self._sparse:
            return 'fused'
        if isinstance(net, BilinearNet) and not self._sparse and net.fused_spec() is not None and \
                fused_kind in (_lib.OPT_SGD, _lib.OPT_ADAGRAD):
            return 'bloom'
        return 'generic'

    def _device(self):
        return next(self._net.parameters()).device

    def fit(self, interactions, verbose=False):
        """Fit the model; repeated calls resume from the current weights and
        optimizer state (explicit.py:173-243)."""
        user_ids = interactions.user_ids
        item_ids = interactions.item_ids

        if not self._initialized:
            self._initialize(interactions)
        if not self._use_cuda:
            raise RuntimeError(_NO_CPU)

        route = self._route()
        device = self._device()
        n = len(user_ids)
        main = torch.cuda.current_stream(device)
        copy_stream = _side_stream(device)
        copy_stream.wait_stream(main)
        with torch.cuda.stream(copy_stream):
            users_dev = _to_device_narrow(user_ids, device)
            items_dev = _to_device_narrow(item_ids, device)
        main.wait_stream(copy_stream)
        users_dev.record_stream(main)
        items_dev.record_stream(main)
        if users_dev.dtype != items_dev.dtype:
            users_dev, items_dev = users_dev.long(), items_dev.long()
        if n:
            umax, imax, umin, imin = torch.stack([users_dev.max(), items_dev.max(), users_dev.min(),
                                                  items_dev.min()]).tolist()        # one sync
            self._check_input(int(umax), int(imax))
            if umin < 0 or imin < 0:
                # the reference fails inside the embedding lookup
                raise IndexError('index out of range in self: negative user or item id')
        if self._n_iter <= 0:
            return
        if interactions.ratings is None:
            # the reference's shuffle(user_ids, item_ids, None) fails the same way (explicit.py:201-204)
            raise TypeError("object of type 'NoneType' has no len()")
        if len(interactions.ratings) != n:
            raise ValueError('All inputs to shuffle must have the same length.')
        if torch.is_tensor(interactions.ratings) and interactions.ratings.is_cuda:
            ratings_dev = interactions.ratings.to(device, torch.float32).contiguous()
        else:
            ratings_dev = torch.from_numpy(np.ascontiguousarray(interactions.ratings, dtype=np.float32)).to(device)

        on_device = DEVICE_SHUFFLE_MIN <= n <= SHUFFLE_DEVICE_MAX and \
            self._random_state.get_state()[0] == 'MT19937'
        pending = (shuffle_begin(n, self._random_state, device), main) if on_device else None

        for epoch_num in range(self._n_iter):
            # shuffle(): the same stream consumption as random_state.shuffle(arange(n))
            # (torch_utils.py:46-47); the gathers run on the device
            if pending is not None:
                handle, stream = pending
                with torch.cuda.stream(stream):
                    order_dev = shuffle_end(handle)
                if stream is not main:
                    main.wait_stream(stream)
                    order_dev.record_stream(main)
                pending = None
            elif on_device:
                order_dev = shuffled_order_device(n, self._random_state, device)
            else:
                order = shuffled_order(n, self._random_state)
                order_dev = torch.from_numpy(order).to(device).long()
            users_t, items_t = permute_ids(order_dev, users_dev, items_dev)
            ratings_t = ratings_dev.index_select(0, order_dev)
            del order_dev

            if route == 'epoch':
                if on_device and epoch_num + 1 < self._n_iter:
                    # nothing else draws from the stream: the next epoch's shuffle runs on the
                    # side stream under this epoch's training steps
                    side = _side_stream(device)
                    side.wait_stream(main)
                    with torch.cuda.stream(side):
                        pending = (shuffle_begin(n, self._random_state, device), side)
                epoch_loss = self._fit_epoch_pipeline(users_t, items_t, ratings_t)
            elif route == 'bloom':
                epoch_loss = self._fit_epoch_bloom_fused(users_t, items_t, ratings_t)
            else:
                epoch_loss = self._fit_epoch_autograd(users_t, items_t, ratings_t, route)

            if verbose:
                print('Epoch {}: loss {}'.format(epoch_num, epoch_loss))

            if np.isnan(epoch_loss) or epoch_loss == 0.0:
                raise ValueError('Degenerate epoch loss: {}'.format(epoch_loss))
        if hasattr(self._optimizer, 'flush'):
            self._optimizer.flush()             # lazy-exact Adam: every row current before fit() returns

    def _fit_epoch_pipeline(self, users, items, ratings):
        """One ``slb_mf_fit_epoch`` call enqueues every minibatch step (fused optimizer,
        compact gradients); returns the mean of the per-batch losses (explicit.py:231,236)."""
        net = self._net
        lib = _lib.load()
        n, B = users.numel(), int(self._batch_size)
        params = (net.user_embeddings.weight, net.item_embeddings.weight, net.user_biases.weight,
                  net.item_biases.weight)
        dev = params[0].device
        n_steps = (n + B - 1) // B
        with torch.no_grad():
            kind, hp, states, adam = _fused_optimizer(self._optimizer, params, n_steps, dev)
            # the planned step runs in its one-term mode (csrc/mf_v2.cuh)
            a, ws, keep = ops.mf_fused_step_args(*params, users, items, None, self._loss, 1, kind, hp, states,
                                                 batch=min(B, n), ratings=ratings, adam=adam,
                                                 planned=implicit.PLANNED_STEP)
            if a.fused_workspace:
                a.plan_stream = _plan_stream(dev).cuda_stream
            losses = torch.empty(n_steps, dtype=torch.float32, device=dev)
            rc = lib.slb_mf_fit_epoch(ctypes.byref(a), ops._ptr(users), ops._ptr(items), None, n,
                                      ops._ptr(losses), ops._stream())
            _lib.check(rc, 'mf_fit_epoch')
            host = losses.cpu().numpy().astype(np.float64)                  # one sync per epoch
            if ops.workspace_error_flag(ws):
                raise ValueError('ids out of range reached the device kernels')
        return float(host.sum() / n_steps)

    def _fit_epoch_bloom_fused(self, users, items, ratings):
        """Hashed-table model with fused SGD / Adagrad: one in-place step per minibatch
        (csrc/mf.cu slb_mf_bloom_train_step with a rating loss), no dense gradient of any table;
        returns the mean of the per-batch losses (explicit.py:231,236)."""
        net, opt = self._net, self._optimizer
        spec = net.fused_spec()
        hp = opt.fused_hparams()
        params = (spec['Wu'], spec['Wi'], net.user_biases.weight, net.item_biases.weight)
        states = [opt.fused_state(p) for p in params] if opt.fused_kind == _lib.OPT_ADAGRAD else None
        losses = []
        for batch_user, batch_item, batch_ratings in minibatch(users, items, ratings, batch_size=self._batch_size):
            losses.append(ops.mf_bloom_train_step_inplace(
                *params, batch_user, batch_item, None, self._loss, 1, spec['user_seeds'], spec['item_seeds'],
                spec['user_pad'], spec['item_pad'], opt.fused_kind, hp['lr'], states, hp['weight_decay'],
                hp['eps'], ratings=batch_ratings))
        host = torch.stack(losses).cpu().numpy().astype(np.float64)        # one sync per epoch
        return float(host.sum() / len(host))

    def _fit_epoch_autograd(self, users, items, ratings, route):
        net = self._net
        epoch_loss = torch.zeros((), dtype=torch.float64, device=users.device)
        minibatch_num = -1
        for minibatch_num, (batch_user, batch_item, batch_ratings) in enumerate(
                minibatch(users, items, ratings, batch_size=self._batch_size)):
            self._optimizer.zero_grad()
            if route == 'fused':
                loss = ops.fused_rating_loss(net.user_embeddings.weight, net.item_embeddings.weight,
                                             net.user_biases.weight, net.item_biases.weight,
                                             batch_user, batch_item, batch_ratings, self._loss)
            else:
                predictions = net(batch_user, batch_item)
                if self._loss == 'poisson':
                    predictions = torch.exp(predictions)
                loss = self._loss_func(batch_ratings, predictions)
            epoch_loss += loss.detach().double()
            loss.backward()
            self._optimizer.step()
        return float(epoch_loss.item()) / (minibatch_num + 1)

    def _predict_device(self, user_ids, item_ids):
        """Predictions for int64 CUDA id tensors, as a float32 CUDA tensor (no host copy)."""
        self._net.train(False)
        with torch.no_grad():
            out = self._net(user_ids, item_ids)
            if self._loss == 'poisson':
                out = torch.exp(out)
            elif self._loss == 'logistic':
                out = torch.sigmoid(out)
        return out.reshape(-1)

    def predict(self, user_ids, item_ids=None):
        """Predicted ratings for (user, item) pairs, or for one user against ``item_ids``
        (all items when None): ``exp`` of the score for poisson, ``sigmoid`` for logistic;
        returns a NumPy array (explicit.py:245-284)."""
        self._check_input(user_ids, item_ids, allow_items_none=True)
        user_ids, item_ids = _predict_process_ids(user_ids, item_ids, self._num_items,
                                                  self._use_cuda)
        return cpu(self._predict_device(user_ids, item_ids)).numpy().flatten()
