"""Sequence representations with the reference's classes, constructor
arguments and parameter names (spotlight/sequence/representations.py:27-596).

``PoolNet``, ``CNNNet``, ``LSTMNet`` and ``MixtureLSTMNet`` run on the kernels of
csrc/seq.cu; all keep the reference's module protocol -- ``user_representation(item_sequences)
-> (all_steps (B, D, S), final (B, D))`` (``MixtureLSTMNet``: ``(B, 2M, D, S)``, ``(B, 2M, D,
1)``) and ``forward(user_representations, targets) -> (B, S)`` -- so they also work with
external training loops and the reference's evaluation code.
"""

import torch
import torch.nn as nn
import torch.nn.functional as F

from spotlight_b200 import ops
from spotlight_b200.layers import BloomEmbedding, ScaledEmbedding, ZeroEmbedding

PADDING_IDX = 0


def _to_iterable(val, num):
    try:
        iter(val)
        return val
    except TypeError:
        return (val,) * num


class _SeqNetBase(nn.Module):
    """Shared scoring head: dot(user representation, target embedding) + bias
    (representations.py:136-144, 444-453)."""

    def _cnn_spec(self):
        return None

    def _lstm_spec(self):
        return None

    def _mixture_spec(self):
        return None

    def _autograd_params(self):
        return (self.item_embeddings.weight,)

    def fusable(self):
        emb = self.item_embeddings
        return (type(emb) is ScaledEmbedding and emb.padding_idx == PADDING_IDX and not emb.sparse
                and emb.embedding_dim % 4 == 0 and emb.embedding_dim <= 512
                and not self.item_biases.sparse)

    def _kernel_limits(self):
        """The representation's own limits of the fused step (dimension, layer shapes)."""
        return self.item_embeddings.embedding_dim <= 512

    def hashed_spec(self):
        """``dict(seeds, padding_idx)`` when the item layer is a ``BloomEmbedding`` the fused sequence
        step can train (padding id 0, dense table, ``D % 4 == 0``, within the net's kernel limits);
        None otherwise."""
        emb = self.item_embeddings
        if not (isinstance(emb, BloomEmbedding) and emb.padding_idx == PADDING_IDX
                and not emb.embeddings.sparse and emb.embedding_dim % 4 == 0 and emb.num_hash_functions >= 1
                and emb.compressed_num_embeddings >= 1 and not self.item_biases.sparse and self._kernel_limits()):
            return None
        return dict(seeds=list(emb._masks), padding_idx=PADDING_IDX)

    def _item_table(self):
        """The item table the fused step trains: the plain weight, or a BloomEmbedding's compressed one."""
        emb = self.item_embeddings
        return emb.embeddings.weight if isinstance(emb, BloomEmbedding) else emb.weight

    def user_representation(self, item_sequences):
        """``(all, final)``: ``all[:, :, t]`` has seen items before ``t``
        (t = 0..S-1), ``final`` has seen the whole sequence."""
        if not self.fusable() or (torch.is_grad_enabled()
                                  and any(p.requires_grad for p in self._autograd_params())):
            # custom / Bloom item layers, or an external training loop that needs
            # autograd through the representation: differentiable composition over
            # this package's embedding op (not the measured path)
            return self._user_representation_autograd(item_sequences)
        rep = ops.seq_representation(self.item_embeddings.weight.detach(),
                                     item_sequences, self._cnn_spec(), lstm=self._lstm_spec())
        rep = rep.permute(0, 2, 1)                      # (B, D, S+1) like the reference
        return rep[:, :, :-1], rep[:, :, -1]

    def forward(self, user_representations, targets):
        dim = self.embedding_dim
        target_embedding = self.item_embeddings(targets)            # (B, S, D) or (B, 1, D)
        target_bias = self.item_biases(targets).reshape(targets.shape)
        if user_representations.dim() == 2:                          # predict: (N, D) x (N, 1)
            dot = (user_representations * target_embedding.reshape(-1, dim)).sum(1)
            return target_bias.reshape(-1) + dot
        dot = (user_representations.permute(0, 2, 1) * target_embedding).sum(2)
        return target_bias + dot


class PoolNet(_SeqNetBase):
    """Average of the embeddings of all items seen so far
    (representations.py:27-144).  Parameters: ``item_embeddings.weight (I, D)``
    with ``padding_idx=0`` and ``item_biases.weight (I, 1)``."""

    def __init__(self, num_items, embedding_dim=32, item_embedding_layer=None, sparse=False):
        super(PoolNet, self).__init__()
        self.embedding_dim = embedding_dim
        self.item_embeddings = (item_embedding_layer if item_embedding_layer is not None
                                else ScaledEmbedding(num_items, embedding_dim,
                                                     padding_idx=PADDING_IDX, sparse=sparse))
        self.item_biases = ZeroEmbedding(num_items, 1, sparse=sparse, padding_idx=PADDING_IDX)

    def _user_representation_autograd(self, item_sequences):
        # prefix mean with the element-wise non-zero count (representations.py:91-114)
        emb = self.item_embeddings(item_sequences).permute(0, 2, 1)          # (B, D, S)
        emb = F.pad(emb, (1, 0))                                             # (B, D, S+1)
        total = torch.cumsum(emb, 2)
        count = torch.cumsum((emb != 0.0).float(), 2)
        rep = total / (count + 1)
        return rep[:, :, :-1], rep[:, :, -1]


class CNNNet(_SeqNetBase):
    """Stacked causal dilated 1-d convolutions (representations.py:261-453).

    Parameters: embeddings/biases as ``PoolNet`` plus ``cnn_{i}.weight
    (D, D, k, 1)`` and ``cnn_{i}.bias (D,)`` -- the reference's ``nn.Conv2d``
    shapes, so ``state_dict``s interchange.  The first layer is left-padded by
    its full receptive field so step t only sees items < t (:394-400).
    """

    def __init__(self, num_items, embedding_dim=32, kernel_width=3, dilation=1, num_layers=1,
                 nonlinearity='tanh', residual_connections=True, sparse=False, benchmark=True,
                 item_embedding_layer=None):
        super(CNNNet, self).__init__()
        self.embedding_dim = embedding_dim
        self.kernel_width = _to_iterable(kernel_width, num_layers)
        self.dilation = _to_iterable(dilation, num_layers)
        if nonlinearity not in ('tanh', 'relu'):
            raise ValueError('Nonlinearity must be one of (tanh, relu)')
        self._nonlinearity_name = nonlinearity
        self.nonlinearity = torch.tanh if nonlinearity == 'tanh' else F.relu
        self.residual_connections = residual_connections
        self.item_embeddings = (item_embedding_layer if item_embedding_layer is not None
                                else ScaledEmbedding(num_items, embedding_dim,
                                                     padding_idx=PADDING_IDX, sparse=sparse))
        self.item_biases = ZeroEmbedding(num_items, 1, sparse=sparse, padding_idx=PADDING_IDX)
        self.cnn_layers = [nn.Conv2d(embedding_dim, embedding_dim, (_kernel_width, 1),
                                     dilation=(_dilation, 1))
                           for (_kernel_width, _dilation) in zip(self.kernel_width, self.dilation)]
        for i, layer in enumerate(self.cnn_layers):
            self.add_module('cnn_{}'.format(i), layer)

    def _user_representation_autograd(self, item_sequences):
        # stacked causal dilated convs (representations.py:385-422)
        emb = self.item_embeddings(item_sequences).permute(0, 2, 1).unsqueeze(3)   # (B, D, S, 1)
        kw, dl = list(self.kernel_width), list(self.dilation)
        rf = kw[0] + (kw[0] - 1) * (dl[0] - 1)
        x = self.nonlinearity(self.cnn_layers[0](F.pad(emb, (0, 0, rf, 0))))
        if self.residual_connections:
            x = x + F.pad(emb, (0, 0, 1, 0))
        for layer, k, d in zip(self.cnn_layers[1:], kw[1:], dl[1:]):
            rf = k + (k - 1) * (d - 1)
            residual = x
            x = self.nonlinearity(layer(F.pad(x, (0, 0, rf - 1, 0))))
            if self.residual_connections:
                x = x + residual
        x = x.squeeze(3)
        return x[:, :, :-1], x[:, :, -1]

    def _cnn_spec(self):
        return dict(kernel_width=[int(k) for k in self.kernel_width][:len(self.cnn_layers)],
                    dilation=[int(d) for d in self.dilation][:len(self.cnn_layers)],
                    nonlinearity=self._nonlinearity_name,
                    residual=bool(self.residual_connections),
                    weights=[layer.weight for layer in self.cnn_layers],
                    biases=[layer.bias for layer in self.cnn_layers])


class LSTMNet(_SeqNetBase):
    """Single-layer LSTM over the left zero-padded item sequence (representations.py:147-258).

    Parameters: embeddings/biases as ``PoolNet`` plus ``lstm.weight_ih_l0``, ``lstm.weight_hh_l0``
    ``(4D, D)`` and ``lstm.bias_ih_l0``, ``lstm.bias_hh_l0`` ``(4D,)`` -- the reference's
    ``nn.LSTM``, which stays the parameter holder, so ``state_dict``s interchange.  On a plain
    item table with ``D <= 256`` the representation runs on the recurrence kernels of
    csrc/seq_lstm.cuh; otherwise (Bloom items, larger ``D``) and whenever autograd needs the
    representation, ``nn.LSTM`` computes it.
    """

    LSTM_MAX_DIM = 256

    def __init__(self, num_items, embedding_dim=32, item_embedding_layer=None, sparse=False):
        super(LSTMNet, self).__init__()
        self.embedding_dim = embedding_dim
        self.item_embeddings = (item_embedding_layer if item_embedding_layer is not None
                                else ScaledEmbedding(num_items, embedding_dim,
                                                     padding_idx=PADDING_IDX, sparse=sparse))
        self.item_biases = ZeroEmbedding(num_items, 1, sparse=sparse, padding_idx=PADDING_IDX)
        self.lstm = nn.LSTM(batch_first=True, input_size=embedding_dim, hidden_size=embedding_dim)

    def fusable(self):
        return super(LSTMNet, self).fusable() and self._kernel_limits()

    def _kernel_limits(self):
        return (self.item_embeddings.embedding_dim <= self.LSTM_MAX_DIM
                and self.lstm.num_layers == 1 and self.lstm.bias and not self.lstm.bidirectional)

    def _autograd_params(self):
        return (self.item_embeddings.weight,) + tuple(self.lstm.parameters())

    def _user_representation_autograd(self, item_sequences):
        emb = self.item_embeddings(item_sequences).permute(0, 2, 1).unsqueeze(3)
        emb = F.pad(emb, (0, 0, 1, 0)).squeeze(3).permute(0, 2, 1)
        out, _ = self.lstm(emb)
        out = out.permute(0, 2, 1)
        return out[:, :, :-1], out[:, :, -1]

    def _lstm_spec(self):
        return dict(w_ih=self.lstm.weight_ih_l0.detach(), w_hh=self.lstm.weight_hh_l0.detach(),
                    b_ih=self.lstm.bias_ih_l0.detach(), b_hh=self.lstm.bias_hh_l0.detach())


class MixtureLSTMNet(_SeqNetBase):
    """Mixture-of-tastes LSTM (representations.py:456-596).

    Parameters: ``LSTMNet``'s plus ``projection.weight (2MD, D, 1)`` and ``projection.bias (2MD,)``,
    the reference's ``nn.Conv1d``, so ``state_dict``s interchange.  ``user_representation`` returns
    the reference's ``(B, 2M, D, S)`` and ``(B, 2M, D, 1)``: blocks 0..M-1 are the taste components,
    M..2M-1 the mixture vectors.  On a plain item table with ``D <= 256`` and ``1 <= M <= 8`` it
    runs on the LSTM kernels and the projection GEMMs of csrc/seq.cu; otherwise, and whenever
    autograd needs the representation, ``nn.LSTM`` and ``nn.Conv1d`` compute it.  ``forward`` is
    the reference's softmax head in torch ops (the fused training step has its own kernel).
    """

    LSTM_MAX_DIM = 256
    MAX_MIXTURES = 8

    def __init__(self, num_items, embedding_dim=32, num_mixtures=4, item_embedding_layer=None,
                 sparse=False):
        super(MixtureLSTMNet, self).__init__()
        self.embedding_dim = embedding_dim
        self.num_mixtures = num_mixtures
        self.item_embeddings = (item_embedding_layer if item_embedding_layer is not None
                                else ScaledEmbedding(num_items, embedding_dim,
                                                     padding_idx=PADDING_IDX, sparse=sparse))
        self.item_biases = ZeroEmbedding(num_items, 1, sparse=sparse, padding_idx=PADDING_IDX)
        self.lstm = nn.LSTM(batch_first=True, input_size=embedding_dim, hidden_size=embedding_dim)
        self.projection = nn.Conv1d(embedding_dim, embedding_dim * self.num_mixtures * 2,
                                    kernel_size=1)

    def fusable(self):
        return super(MixtureLSTMNet, self).fusable() and self._kernel_limits()

    def _kernel_limits(self):
        p = self.projection
        return (self.item_embeddings.embedding_dim <= self.LSTM_MAX_DIM
                and 1 <= self.num_mixtures <= self.MAX_MIXTURES
                and self.lstm.num_layers == 1 and self.lstm.bias and not self.lstm.bidirectional
                and type(p) is nn.Conv1d and p.bias is not None and p.kernel_size == (1,)
                and p.groups == 1 and p.stride == (1,) and p.padding == (0,) and p.dilation == (1,))

    def _autograd_params(self):
        return ((self.item_embeddings.weight,) + tuple(self.lstm.parameters())
                + tuple(self.projection.parameters()))

    def _lstm_spec(self):
        return dict(w_ih=self.lstm.weight_ih_l0.detach(), w_hh=self.lstm.weight_hh_l0.detach(),
                    b_ih=self.lstm.bias_ih_l0.detach(), b_hh=self.lstm.bias_hh_l0.detach())

    def _mixture_spec(self):
        return dict(num_mixtures=int(self.num_mixtures), w=self.projection.weight.detach(),
                    b=self.projection.bias.detach())

    def user_representation(self, item_sequences):
        if not self.fusable() or (torch.is_grad_enabled()
                                  and any(p.requires_grad for p in self._autograd_params())):
            return self._user_representation_autograd(item_sequences)
        rep = ops.seq_representation(self.item_embeddings.weight.detach(), item_sequences, None,
                                     lstm=self._lstm_spec(), mixture=self._mixture_spec())
        B, T = rep.shape[0], rep.shape[1]
        rep = rep.view(B, T, 2 * self.num_mixtures, self.embedding_dim).permute(0, 2, 3, 1)
        return rep[:, :, :, :-1], rep[:, :, :, -1:]

    def _user_representation_autograd(self, item_sequences):
        batch_size, sequence_length = item_sequences.size()
        emb = self.item_embeddings(item_sequences).permute(0, 2, 1).unsqueeze(3)
        emb = F.pad(emb, (0, 0, 1, 0)).squeeze(3).permute(0, 2, 1)
        out, _ = self.lstm(emb)
        out = self.projection(out.permute(0, 2, 1))
        out = out.view(batch_size, self.num_mixtures * 2, self.embedding_dim, sequence_length + 1)
        return out[:, :, :, :-1], out[:, :, :, -1:]

    def forward(self, user_representations, targets):
        user_components = user_representations[:, :self.num_mixtures]
        mixture_vectors = user_representations[:, self.num_mixtures:]
        target_embedding = self.item_embeddings(targets).permute(0, 2, 1)
        target_bias = self.item_biases(targets).squeeze(-1)
        mixture_weights = (mixture_vectors * target_embedding.unsqueeze(1).expand_as(user_components))
        mixture_weights = F.softmax(mixture_weights.sum(2), 1).unsqueeze(2).expand_as(user_components)
        weighted = (mixture_weights * user_components).sum(1)
        dot = (weighted * target_embedding).sum(1)
        if dot.dim() > target_bias.dim():
            dot = dot.squeeze(-1)
        return target_bias.reshape(dot.shape) + dot
