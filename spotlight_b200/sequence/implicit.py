"""Implicit-feedback sequence model with the reference's estimator API
(spotlight/sequence/implicit.py:29-331): same constructor arguments,
``fit(interactions, verbose)``, ``predict(sequences, item_ids=None)``.

``fit`` routes
  fused    PoolNet / CNNNet / LSTMNet (D <= 256) / MixtureLSTMNet (D <= 256, at most 8
           mixtures) on a plain ``ScaledEmbedding(padding_idx=0)``: one C
           call per minibatch runs representation, scoring, masked loss and the
           whole backward (deterministic segmented scatter into the embedding
           gradient); the gradients are handed to whatever ``torch.optim``
           optimizer the model holds.
  fused_hashed
           the same four nets on a ``BloomEmbedding(padding_idx=0)`` item layer (dense table,
           within each net's fused limits) trained with ``optim.fused_sgd`` / ``fused_adagrad`` /
           ``fused_adam``: the same C call, with items summed from their hashed rows, and the
           compressed table and the biases updated in place by the row-wise optimizer.

With ``optim.fused_adam`` (row-wise lazy-exact Adam) on either fused route the C call applies
Adam to the item table and bias in place (no dense (num_items, D) gradient, no sweep over the
table); ``optimizer.step()`` then takes the same Adam step on the other parameters, and ``fit()``
flushes the pending steps of every row before it returns.
  generic  any other representation (custom, Bloom-embedded under a ``torch.optim``
           optimizer): the reference's loop shape over this package's gather and loss ops.
"""

import numpy as np
import torch
import torch.optim as optim

from spotlight_b200 import _lib, ops
from spotlight_b200.helpers import _repr_model
from spotlight_b200.losses import adaptive_hinge_loss, bpr_loss, hinge_loss, pointwise_loss
from spotlight_b200.rng import SHUFFLE_DEVICE_MAX, shuffled_order_device
from spotlight_b200.sampling import sample_items
from spotlight_b200.sequence.representations import (PADDING_IDX, CNNNet, LSTMNet,
                                                     MixtureLSTMNet, PoolNet)
from spotlight_b200.torch_utils import cpu, gpu, minibatch, set_seed, shuffled_order

DEVICE_SHUFFLE_MIN = 1 << 17        # as factorization/implicit.py: a speed knob, both paths are bit-exact

_NO_CPU = ('spotlight_b200 runs the fit() hot path in sm_90a CUDA kernels and has no CPU '
           'route; construct the model with use_cuda=True.')


class ImplicitSequenceModel(object):
    """Next-item prediction from interaction sequences.

    Parameters (identical to the reference, implicit.py:85-97): ``loss`` in
    ('pointwise', 'bpr', 'hinge', 'adaptive_hinge'); ``representation`` in
    ('pooling', 'cnn', 'lstm', 'mixture') or a module; ``embedding_dim, n_iter,
    batch_size, l2, learning_rate, optimizer_func, use_cuda, sparse,
    random_state, num_negative_samples``.
    """

    def __init__(self, loss='pointwise', representation='pooling', embedding_dim=32, n_iter=10,
                 batch_size=256, l2=0.0, learning_rate=1e-2, optimizer_func=None, use_cuda=False,
                 sparse=False, random_state=None, num_negative_samples=5):

        assert loss in ('pointwise', 'bpr', 'hinge', 'adaptive_hinge')
        if isinstance(representation, str):
            assert representation in ('pooling', 'cnn', 'lstm', 'mixture')

        self._loss = loss
        self._representation = representation
        self._embedding_dim = embedding_dim
        self._n_iter = n_iter
        self._learning_rate = learning_rate
        self._batch_size = batch_size
        self._l2 = l2
        self._use_cuda = use_cuda
        self._sparse = sparse
        self._optimizer_func = optimizer_func
        self._random_state = random_state or np.random.RandomState()
        self._num_negative_samples = num_negative_samples

        self._num_items = None
        self._net = None
        self._optimizer = None
        self._loss_func = None

        set_seed(self._random_state.randint(-10**8, 10**8), cuda=self._use_cuda)

    def __repr__(self):
        return _repr_model(self)

    @property
    def _initialized(self):
        return self._net is not None

    def _initialize(self, interactions):
        if not self._use_cuda:
            raise RuntimeError(_NO_CPU)
        self._num_items = interactions.num_items
        builders = {'pooling': PoolNet, 'cnn': CNNNet, 'lstm': LSTMNet, 'mixture': MixtureLSTMNet}
        if isinstance(self._representation, str):
            self._net = builders[self._representation](self._num_items, self._embedding_dim,
                                                       sparse=self._sparse)
        else:
            self._net = self._representation
        self._net = gpu(self._net, self._use_cuda)

        if self._optimizer_func is None:
            self._optimizer = optim.Adam(self._net.parameters(), weight_decay=self._l2,
                                         lr=self._learning_rate)
        else:
            self._optimizer = self._optimizer_func(self._net.parameters())

        self._loss_func = {'pointwise': pointwise_loss, 'bpr': bpr_loss, 'hinge': hinge_loss,
                           'adaptive_hinge': adaptive_hinge_loss}[self._loss]

    def _check_input(self, item_ids):
        item_id_max = item_ids if isinstance(item_ids, int) else item_ids.max()
        if item_id_max >= self._num_items:
            raise ValueError('Maximum item id greater than number of items in model.')

    def _n_neg(self):
        return self._num_negative_samples if self._loss == 'adaptive_hinge' else 1

    def _route(self):
        net = self._net
        if isinstance(net, (PoolNet, CNNNet, LSTMNet, MixtureLSTMNet)) and not self._sparse:
            if net.fusable():
                return 'fused'
            # a hashed table has no dense gradient to hand to torch.optim: row-wise optimizers only
            if net.hashed_spec() is not None and \
                    getattr(self._optimizer, 'fused_kind', None) in (_lib.OPT_SGD, _lib.OPT_ADAGRAD, _lib.OPT_ADAM):
                return 'fused_hashed'
        return 'generic'

    def fit(self, interactions, verbose=False):
        """Fit the model; repeated calls resume (implicit.py:193-264)."""
        on_device = torch.is_tensor(interactions.sequences) and interactions.sequences.is_cuda
        sequences = interactions.sequences if on_device else interactions.sequences.astype(np.int64)

        if not self._initialized:
            self._initialize(interactions)
        if not self._use_cuda:
            raise RuntimeError(_NO_CPU)

        self._check_input(sequences)
        route = self._route()
        n_neg = self._n_neg()
        device = next(self._net.parameters()).device

        # the sequences go to the device once per fit(); every epoch permutes the resident rows
        # (cumulatively, as the reference's `sequences = sequences[shuffle_indices]` does,
        # implicit.py:217-220) instead of re-indexing on the host and re-uploading
        if on_device:       # a device SequenceInteractions (to_sequence of CUDA interactions) stays there
            sequences_tensor = sequences.to(device, torch.int64).contiguous()
        else:
            sequences_tensor = gpu(torch.from_numpy(np.ascontiguousarray(sequences)), self._use_cuda)
        n_seq = len(sequences)

        for epoch_num in range(self._n_iter):
            if DEVICE_SHUFFLE_MIN <= n_seq <= SHUFFLE_DEVICE_MAX and \
                    self._random_state.get_state()[0] == 'MT19937':
                order = shuffled_order_device(n_seq, self._random_state, device)
            else:
                order = torch.from_numpy(shuffled_order(n_seq, self._random_state)).to(device).long()
            sequences_tensor = sequences_tensor.index_select(0, order)
            del order
            S = sequences_tensor.shape[1]
            # Per-minibatch draws of shape (n*B, S) (implicit.py:268-271, 283-285)
            # concatenate to one stream-equivalent draw over the epoch.
            negatives = sample_items(self._num_items, (n_seq * n_neg, S),
                                     random_state=self._random_state, device=device)

            epoch_loss = torch.zeros((), dtype=torch.float64, device=device)
            lo = 0
            minibatch_num = -1
            for minibatch_num, batch_sequence in enumerate(
                    minibatch(sequences_tensor, batch_size=self._batch_size)):
                B = batch_sequence.shape[0]
                batch_neg = negatives[lo * n_neg:(lo + B) * n_neg]      # rows k*B + b
                lo += B
                self._optimizer.zero_grad()
                if route in ('fused', 'fused_hashed'):
                    loss = self._fused_step(batch_sequence, batch_neg, n_neg)
                else:
                    loss = self._generic_step(batch_sequence, batch_neg, n_neg)
                    loss.backward()
                epoch_loss += loss.detach().double()
                self._optimizer.step()

            epoch_loss = float(epoch_loss.item()) / (minibatch_num + 1)

            if verbose:
                print('Epoch {}: loss {}'.format(epoch_num, epoch_loss))

            if np.isnan(epoch_loss) or epoch_loss == 0.0:
                raise ValueError('Degenerate epoch loss: {}'.format(epoch_loss))
        if hasattr(self._optimizer, 'flush'):
            self._optimizer.flush()             # lazy-exact Adam: every row current before fit() returns

    def _fused_step(self, batch_sequence, batch_neg, n_neg):
        net = self._net
        spec = net._cnn_spec()
        lstm = net._lstm_spec()
        mixture = net._mixture_spec()
        fused = None
        opt = self._optimizer
        kind = getattr(opt, 'fused_kind', None)
        item_hash = net.hashed_spec()
        table = net._item_table()
        if kind in (_lib.OPT_SGD, _lib.OPT_ADAGRAD):
            # row-wise optimizer inside the step (spotlight_b200.optim): the item table and its bias
            # are updated in place by the gradient kernel, no dense (num_items, D) gradient exists;
            # optimizer.step() below then only sees the (tiny) conv parameters
            hp = opt.fused_hparams()
            fused = dict(kind=kind, lr=hp['lr'], weight_decay=hp['weight_decay'], eps=hp['eps'],
                         state_E=opt.fused_state(table),
                         state_bias=opt.fused_state(net.item_biases.weight))
        elif kind == _lib.OPT_ADAM:
            # lazy-exact Adam inside the step, at step t = steps taken + 1; optimizer.step() below
            # counts t and applies it to the parameters that carry a .grad (not the item table and bias).
            # A plain table's bias shares the rows' `last`; a hashed table and its id-indexed bias have their own.
            hp = opt.fused_hparams()
            hashed = item_hash is not None
            m, v, last = opt.fused_states(table, own_last=hashed)
            bm, bv, blast = opt.fused_states(net.item_biases.weight, own_last=hashed)
            t = opt.steps_taken + 1
            fused = dict(kind=kind, lr=hp['lr'], weight_decay=hp['weight_decay'], eps=hp['eps'],
                         beta1=hp['beta1'], beta2=hp['beta2'], state_E=m, state_bias=bm, state2_E=v, state2_bias=bv,
                         last_E=last, last_bias=blast if hashed else None, sched=opt.schedule(t, table.device), step=t)
        with torch.no_grad():
            out = ops.seq_train_step(table, net.item_biases.weight,
                                     batch_sequence, batch_neg, self._loss, n_neg, spec, fused=fused,
                                     lstm=lstm, mixture=mixture, item_hash=item_hash)
        table.grad = out['dE']
        net.item_biases.weight.grad = out['dbias']
        if spec is not None:
            for layer, dw, db in zip(net.cnn_layers, out['dconv_w'], out['dconv_b']):
                layer.weight.grad = dw
                layer.bias.grad = db
        if lstm is not None:
            g = out['dlstm']
            net.lstm.weight_ih_l0.grad, net.lstm.weight_hh_l0.grad = g['w_ih'], g['w_hh']
            net.lstm.bias_ih_l0.grad, net.lstm.bias_hh_l0.grad = g['b_ih'], g['b_hh']
        if mixture is not None:
            net.projection.weight.grad = out['dmix']['w']
            net.projection.bias.grad = out['dmix']['b']
        return out['loss']

    def _generic_step(self, batch_sequence, batch_neg, n_neg):
        net = self._net
        B, S = batch_sequence.shape
        user_representation, _ = net.user_representation(batch_sequence)
        positive_prediction = net(user_representation, batch_sequence)
        if self._loss == 'adaptive_hinge':
            size = (n_neg,) + (1,) * (user_representation.dim() - 1)
            negative_prediction = net(user_representation.repeat(*size),
                                      batch_neg).view(n_neg, B, S)
        else:
            negative_prediction = net(user_representation, batch_neg)
        return self._loss_func(positive_prediction, negative_prediction,
                               mask=(batch_sequence != PADDING_IDX))

    def predict(self, sequences, item_ids=None):
        """Scores of ``item_ids`` (all items when None) as the next item of one
        sequence (implicit.py:288-331)."""
        self._net.train(False)
        sequences = np.atleast_2d(sequences)
        if item_ids is None:
            item_ids = np.arange(self._num_items).reshape(-1, 1)
        self._check_input(item_ids)
        self._check_input(sequences)

        sequences = torch.from_numpy(sequences.astype(np.int64).reshape(1, -1))
        item_ids = torch.from_numpy(np.asarray(item_ids).astype(np.int64).reshape(-1, 1))
        sequence_var = gpu(sequences, self._use_cuda)
        item_var = gpu(item_ids, self._use_cuda)

        with torch.no_grad():
            _, sequence_representations = self._net.user_representation(sequence_var)
            size = (len(item_var),) + sequence_representations.size()[1:]
            out = self._net(sequence_representations.expand(*size), item_var)
        return cpu(out).detach().numpy().flatten()
