"""Multi-GPU training step for the matrix-factorisation hot path (SURVEY §8e).

The reference has no distributed code at all; this is the new design the north
star asks for.  One process per GPU (``torch.distributed``, NCCL over
NVLink/NVSwitch):

* **Partitioning.**  User rows (embedding, bias, optimizer state) are owned by
  contiguous user-id ranges; every interaction of the global minibatch is
  processed by the rank that owns its user, so user gathers and the in-place
  user update are always local.  Item rows are sharded by contiguous index range
  (``owner = id // ceil(num_items / world)``).
* **Forward exchange.**  Each rank buckets the distinct item ids of its local
  batch by owner (``unique_bucket``: one counting pass + scan, ids come out
  ascending = grouped by owner), sends the request lists with an all-to-all,
  owners gather rows + biases from their shard and a second all-to-all returns
  them: each needed row crosses NVLink once per rank per step regardless of how
  often the batch uses it.
* **Local step.**  The fused kernels run on (local user shard, received row
  cache) with the batch's item ids remapped onto the cache; loss and gradients
  are normalised by the *global* batch size so the step equals the single-GPU
  step of the concatenated batch.  User rows are updated in place.
* **Backward exchange.**  The per-distinct-row item gradients (already reduced
  locally, deterministically) travel back with the mirrored all-to-all; each
  owner sums the contributions of its peers in rank order (segmented, no float
  atomics) and applies the row-wise Adagrad update to its shard.
* **Loss.**  One scalar all-reduce.

All collectives are ``all_to_all_single`` / ``all_reduce`` of
``torch.distributed``; the compute pieces are the product's CUDA kernels
(:class:`GpuBackend`).  The routing logic is backend-agnostic so it can be
exercised on CPU with ``gloo`` (tests/test_sharded_cpu.py injects a NumPy
backend there; this module itself never imports the oracle).
"""

import ctypes

import numpy as np
import torch
import torch.distributed as dist

from spotlight_b200 import _lib, ops


class ShardPlan(object):
    """Contiguous range partition of users and items over ``world`` ranks."""

    def __init__(self, num_users, num_items, world):
        self.num_users, self.num_items, self.world = int(num_users), int(num_items), int(world)
        self.uchunk = -(-self.num_users // self.world)
        self.ichunk = -(-self.num_items // self.world)

    def user_range(self, rank):
        lo = min(rank * self.uchunk, self.num_users)
        return lo, min(lo + self.uchunk, self.num_users)

    def item_range(self, rank):
        lo = min(rank * self.ichunk, self.num_items)
        return lo, min(lo + self.ichunk, self.num_items)

    def user_owner(self, user_ids):
        return user_ids // self.uchunk


def _users_only_args(st, W, b, users, items, negs, loss, n_neg, dWi, dbi, norm_batch, batch=None, t=None,
                     workspaces=None):
    """A filled ``slb_mf_step_args`` in the step's users-only mode: the user shard's rows and biases
    take their row-wise Adagrad step in place (under ``st.opt`` lazy-exact Adam step ``t``: the
    referenced user rows catch up through t - 1, the touched ones take step t), while the item rows
    ``W`` / ``b`` stay as they are and their gradient goes to the zeroed dense ``dWi`` / ``dbi``
    for the owners; loss and gradients are normalised by ``norm_batch``.  The planned step
    (csrc/mf_v2.cuh) gets the fused workspace where ops.v2_eligible allows.

    ``workspaces``: the (step, fused) workspaces of the stream the step runs on, for a caller that
    fills the arguments on another stream (``ops.workspace`` is per stream); by default the current
    stream's, the fused one only for the planned step.  The caller sets ``loss_out`` and launches."""
    dev = st.Wu.device
    a = ops.mf_step_args(st.Wu, W, st.bu, b, users, items, negs, loss, n_neg, batch=batch)
    a.grad_mode = _lib.GRAD_DENSE
    a.dWi, a.dbi = dWi.data_ptr(), dbi.data_ptr()
    a.norm_batch, a.opt_users_only = int(norm_batch), 1
    if st.opt is not None:
        hp = st.opt.fused_hparams()
        a.opt, a.lr, a.weight_decay, a.eps = _lib.OPT_ADAM, hp['lr'], hp['weight_decay'], hp['eps']
        a.state_Wu, a.state_bu = st.mWu.data_ptr(), st.mbu.data_ptr()
        a.state2_Wu, a.state2_bu, a.last_u = st.vWu.data_ptr(), st.vbu.data_ptr(), st.last_u.data_ptr()
        ops._adam_scalars(a, hp['beta1'], hp['beta2'], st.opt.schedule(t, dev), t)
    else:
        a.opt, a.lr, a.weight_decay, a.eps = _lib.OPT_ADAGRAD, st.lr, 0.0, st.eps
        a.state_Wu, a.state_bu = st.sWu.data_ptr(), st.sbu.data_ptr()
    ws, fws = workspaces if workspaces is not None else ops._mf_workspaces(a, dev)
    a.workspace, a.workspace_bytes = ws.data_ptr(), ws.numel()
    if fws is not None and ops.v2_eligible(a):
        a.fused_workspace, a.fused_workspace_bytes = fws.data_ptr(), fws.numel()
    return a


class GpuBackend(object):
    """The compute pieces of the sharded step on the product's CUDA kernels."""

    def __init__(self, device):
        self.device = torch.device(device)

    def unique_bucket(self, ids, rows, chunk, nparts):
        """distinct ids ascending, inverse map, and per-owner boundaries (host list).  An id
        outside [0, rows) raises ValueError (the kernels would count and train it as row 0)."""
        lib = _lib.load()
        ids = ids.contiguous()
        n = ids.numel()
        uniq = torch.empty(min(n, rows), dtype=torch.int64, device=ids.device)
        inverse = torch.empty(n, dtype=torch.int64, device=ids.device)
        # nparts + 1 owner boundaries, the distinct count, then the workspace's id-range error word
        counts = torch.empty(nparts + 3, dtype=torch.int64, device=ids.device)
        ws = ops.workspace('uq%d' % rows, lib.slb_unique_workspace_bytes(n, rows), ids.device)
        rc = lib.slb_unique_bucket(ops._ptr(ids), n, rows, chunk, nparts, ops._ptr(uniq),
                                   ops._ptr(inverse), ops._ptr(counts), ops._ptr(ws), ws.numel(),
                                   ops._stream())
        _lib.check(rc, 'unique_bucket')
        err = ops.workspace_error_word(ws)
        counts[nparts + 2:].copy_(err)
        host = counts.tolist()                       # the step's one bucketing sync
        if host[nparts + 2]:
            err.zero_()                              # the cached workspace serves the next call clean
            raise ValueError('unique_bucket: an id outside [0, %d) reached the row exchange' % rows)
        return uniq[:host[nparts + 1]], inverse, host[:nparts + 1]

    def gather(self, W, b, local_ids):
        rows = ops.embedding(W, local_ids, [], -1)
        bias = ops.embedding(b.reshape(-1, 1), local_ids, [], -1).reshape(-1)
        return rows, bias

    def local_step(self, st, cache_rows, cache_bias, n_cache, users_local, pos_idx, neg_idx,
                   loss, global_batch, n_neg=1, t=None):
        """Fused forward/backward on (user shard, row cache).  Updates the user
        shard in place (row-wise Adagrad; under ``st.opt``, lazy-exact Adam step ``t``); returns
        (loss share, d cache rows, d cache bias)."""
        cap, D = cache_rows.shape
        loss_out = torch.empty(1, dtype=torch.float32, device=self.device)
        dWi = torch.zeros((cap, D), dtype=torch.float32, device=self.device)
        dbi = torch.zeros(cap, dtype=torch.float32, device=self.device)
        a = _users_only_args(st, cache_rows, cache_bias, users_local, pos_idx, neg_idx, loss, n_neg, dWi, dbi,
                             global_batch, t=t)
        a.loss_out = loss_out.data_ptr()
        _lib.check(_lib.load().slb_mf_train_step(ctypes.byref(a), ops._stream()), 'mf_train_step')
        return loss_out.reshape(()), dWi[:n_cache], dbi[:n_cache]

    def owner_update(self, st, local_ids, g_rows, g_bias):
        """Sum the peers' gradient rows per shard row (rank order, deterministic)
        and apply Adagrad to those rows of the item shard and its bias only."""
        R = local_ids.numel()
        if R == 0:
            return
        lib = _lib.load()
        rows, D = st.Wi.shape
        ids = local_ids.contiguous().long()
        g_rows, g_bias = g_rows.contiguous(), g_bias.reshape(-1).contiguous()
        ws = ops.workspace('shrows%d' % rows, lib.slb_shard_rows_workspace_bytes(R, rows), self.device)
        _lib.check(lib.slb_shard_rows_adagrad(ops._ptr(ids), ops._ptr(g_rows), ops._ptr(g_bias), R,
                                              ops._ptr(st.Wi), ops._ptr(st.sWi), ops._ptr(st.bi), ops._ptr(st.sbi),
                                              rows, D, st.lr, st.eps, ops._ptr(ws), ws.numel(), ops._stream()),
                   'shard_rows_adagrad')

    def _adam_tables(self, st, t, users=False):
        """The item shard (the user shard: ``users``), its bias and their lazy-exact Adam state, with
        step t's scalars (the arguments the row-wise Adam entries share after their ids)."""
        hp = st.opt.fused_hparams()
        W, m, v, b, bm, bv, last = self._adam_pair(st, users)
        rows, D = W.shape
        return (ops._ptr(W), ops._ptr(m), ops._ptr(v), ops._ptr(b), ops._ptr(bm), ops._ptr(bv), ops._ptr(last),
                rows, D, ops._ptr(st.opt.schedule(t, self.device)), t,
                hp['beta1'], hp['beta2'], 1.0 - hp['beta1'], 1.0 - hp['beta2'], hp['eps'], hp['weight_decay'])

    def owner_adam_catch_up(self, st, local_ids, t):
        """Lazy-exact Adam before the gather of step t: the requested rows of the item shard and
        their biases replay the steps they missed, through t - 1."""
        R = local_ids.numel()
        if R == 0:
            return
        ids = local_ids.contiguous().long()
        _lib.check(_lib.load().slb_shard_rows_adam_catch_up(ops._ptr(ids), R, *self._adam_tables(st, t),
                                                            ops._stream()), 'shard_rows_adam_catch_up')

    def user_adam_catch_up(self, st, user_ids, t):
        """Lazy-exact Adam before adaptive hinge scores step t: the user rows ``user_ids`` (local,
        repeats allowed) and their biases replay the steps they missed, through t - 1."""
        R = user_ids.numel()
        if R == 0:
            return
        ids = user_ids.contiguous().long()
        _lib.check(_lib.load().slb_shard_rows_adam_catch_up(ops._ptr(ids), R, *self._adam_tables(st, t, True),
                                                            ops._stream()), 'shard_rows_adam_catch_up')

    def owner_adam_update(self, st, local_ids, g_rows, g_bias, t):
        """Sum the peers' gradient rows per shard row (rank order, deterministic) and take Adam
        step t on those rows of the item shard and their biases only."""
        R = local_ids.numel()
        if R == 0:
            return
        lib = _lib.load()
        ids = local_ids.contiguous().long()
        g_rows, g_bias = g_rows.contiguous(), g_bias.reshape(-1).contiguous()
        ws = ops.workspace('shrows%d' % st.Wi.shape[0], lib.slb_shard_rows_workspace_bytes(R, st.Wi.shape[0]),
                           self.device)
        _lib.check(lib.slb_shard_rows_adam(ops._ptr(ids), ops._ptr(g_rows), ops._ptr(g_bias), R,
                                           *self._adam_tables(st, t), ops._ptr(ws), ws.numel(), ops._stream()),
                   'shard_rows_adam')

    def _adam_pair(self, st, users):
        """The user shard (``users``) or the item shard, with its bias and their Adam state."""
        if users:
            return st.Wu, st.mWu, st.vWu, st.bu, st.mbu, st.vbu, st.last_u
        return st.Wi, st.mWi, st.vWi, st.bi, st.mbi, st.vbi, st.last

    def _adam_scalars(self, st):
        hp = st.opt.fused_hparams()
        return (hp['beta1'], hp['beta2'], 1.0 - hp['beta1'], 1.0 - hp['beta2'], hp['eps'], hp['weight_decay'],
                ops._stream())

    def owner_adam_catch_up_shard(self, st, upto):
        """Every row of the item shard and its bias current through step ``upto``: before the dense
        exchange gathers the whole shard."""
        W, m, v, b, bm, bv, last = self._adam_pair(st, False)
        if upto < 1:
            return
        sched = st.opt.schedule(upto, self.device)
        _lib.check(_lib.load().slb_adam_flush(ops._ptr(W), ops._ptr(m), ops._ptr(v), ops._ptr(b), ops._ptr(bm),
                                              ops._ptr(bv), ops._ptr(last), W.shape[0], W.shape[1], ops._ptr(sched),
                                              upto, *self._adam_scalars(st)), 'adam_flush')

    def adam_dense(self, st, users, g, g_bias, t):
        """Dense Adam step t on the user shard (``users``) or the item shard and its bias: every
        row replays its pending steps, then takes step t with its gradient row, zero rows included."""
        W, m, v, b, bm, bv, last = self._adam_pair(st, users)
        sched = st.opt.schedule(t, self.device)
        g, g_bias = g.contiguous(), g_bias.reshape(-1).contiguous()
        _lib.check(_lib.load().slb_adam_dense(ops._ptr(W), ops._ptr(m), ops._ptr(v), ops._ptr(b), ops._ptr(bm),
                                              ops._ptr(bv), ops._ptr(last), ops._ptr(g), ops._ptr(g_bias),
                                              W.shape[0], W.shape[1], ops._ptr(sched), t,
                                              *self._adam_scalars(st)), 'adam_dense')

    def owner_adam_flush(self, st):
        """Every row of the item shard and its bias current for the steps taken (FusedAdam.flush);
        an empty item range has nothing to flush."""
        if st.Wi.shape[0]:
            st.opt.flush()

    # ---- hashed item table (BloomEmbedding, config 4) ----
    def bloom_local_step(self, st, W_full, users_local, items, negs, loss, global_batch, t=None):
        """Users-only hashed step on (local user shard, full hashed item table, replicated item
        bias): the user rows and user biases take their step in place (row-wise Adagrad; under
        ``st.opt``, lazy-exact Adam step ``t``), O(batch).  Returns (loss share, None, dWi, None, item
        bias pairs), dWi padded to the whole-table exchange's ``world * mchunk`` rows."""
        D = W_full.shape[1]
        dW = torch.zeros((st.world * st.mchunk, D), dtype=torch.float32, device=self.device)
        if st.opt is None:
            uo = dict(opt=_lib.OPT_ADAGRAD, lr=st.lr, eps=st.eps, states=(st.sWu, st.sbu))
        else:
            hp = st.opt.fused_hparams()
            uo = dict(opt=_lib.OPT_ADAM, lr=hp['lr'], eps=hp['eps'], weight_decay=hp['weight_decay'],
                      beta1=hp['beta1'], beta2=hp['beta2'], sched=st.opt.schedule(t, self.device), step=t,
                      states=((st.mWu, st.vWu, st.last_u), (st.mbu, st.vbu), (st.mbi, st.vbi, st.last_bi)))
        out = ops.mf_bloom_step_pairs(st.Wu, W_full, st.bu2, st.bi2, users_local, items, negs, loss,
                                      st.item_seeds, 0, norm_batch=global_batch, users_only=uo, dWi=dW[:st.M])
        return out[0], None, dW, None, out[4]

    def bloom_adam_dense(self, st, g_shard, t):
        """Dense Adam step t on this rank's hashed shard: every row current through t afterwards."""
        g_shard = g_shard.contiguous()
        _lib.check(_lib.load().slb_adam_dense_table(
            ops._ptr(st.Wi), ops._ptr(st.mWi), ops._ptr(st.vWi), ops._ptr(st.last_i), ops._ptr(g_shard),
            st.Wi.shape[0], st.Wi.shape[1], ops._ptr(st.opt.schedule(t, self.device)), t,
            *self._adam_scalars(st)), 'adam_dense_table')

    def bloom_bias_adam(self, st, ids, g, t):
        """Adam step t of the replicated item bias from the all-gathered (id, g) pairs."""
        hp = st.opt.fused_hparams()
        ops.bias_sparse_adam(ids, g, st.bi, st.mbi, st.vbi, st.last_bi, st.opt.schedule(t, self.device), t,
                             hp['beta1'], hp['beta2'], hp['eps'], hp['weight_decay'])

    def adagrad_dense(self, W, S, G, lr, eps):
        _lib.check(_lib.load().slb_adagrad_dense(ops._ptr(W), ops._ptr(S), ops._ptr(G.contiguous()), W.numel(),
                                                 lr, eps, ops._stream()), 'adagrad_dense')

    def bias_sparse_adagrad(self, ids, g, bias, state, lr, eps):
        ops.bias_sparse_apply(ids, g, bias, state, _lib.OPT_ADAGRAD, lr, 0.0, eps)

    # ---- adaptive hinge: scores, loss and score gradients as separate calls ----
    def scores(self, st, cache_rows, cache_bias, u_idx, i_idx):
        return ops.mf_scores(st.Wu, cache_rows, st.bu.reshape(-1, 1), cache_bias.reshape(-1, 1), u_idx, i_idx)

    def adaptive_loss(self, pos, negmat):
        """(mean hinge against the column maxima, d/dpos, d/dneg) -- losses.py:127-166."""
        return ops.pairwise_loss(pos, negmat, None, _lib.LOSS_KIND['adaptive_hinge'])

    def scores_backward(self, st, cache_rows, g, u_idx, i_idx):
        return ops.mf_scores_backward(g, st.Wu, cache_rows, u_idx, i_idx)

    # ---- epoch-level pieces of fit() (all ranks compute the same global stream) ----
    def to_device(self, ids):
        arr = np.ascontiguousarray(ids)
        if arr.dtype not in (np.int32, np.int64):
            arr = arr.astype(np.int64)
        host = torch.from_numpy(arr)
        return host.to(self.device, non_blocking=host.is_pinned())

    def shuffled_order(self, n, random_state):
        from spotlight_b200 import rng
        from spotlight_b200.torch_utils import shuffled_order
        if n >= (1 << 17) and n <= rng.SHUFFLE_DEVICE_MAX:
            return rng.shuffled_order_device(n, random_state, self.device)
        return torch.from_numpy(shuffled_order(n, random_state)).to(self.device).long()

    def permute(self, order, users, items):
        from spotlight_b200 import rng
        return rng.permute_ids(order, users, items)

    def sample(self, num_items, count, random_state):
        from spotlight_b200.sampling import sample_items
        return sample_items(num_items, count, random_state=random_state, device=self.device)

    def upload_sharded(self, ids, rank, world, group=None):
        """Host ids -> the full array on this device with 1/world of the PCIe traffic: every
        rank holds the same host array (single-process semantics), uploads only its slice and
        the slices meet over NVLink (all-gather)."""
        arr = np.ascontiguousarray(ids)
        if arr.dtype not in (np.int32, np.int64):
            arr = arr.astype(np.int64)
        n = arr.shape[0]
        if world == 1 or n < (1 << 16):
            return self.to_device(arr)
        per = -(-n // world)
        lo, hi = min(rank * per, n), min((rank + 1) * per, n)
        host = torch.from_numpy(arr[lo:hi])
        part = torch.zeros(per, dtype=host.dtype, device=self.device)
        part[:hi - lo].copy_(host, non_blocking=host.is_pinned())
        full = torch.empty(per * world, dtype=host.dtype, device=self.device)
        dist.all_gather_into_tensor(full, part, group=group)
        return full[:n]

    def epoch_sampler(self, num_items, random_state, total):
        """Chunked global negative stream on a side stream (device-chained draws, one
        hand-back): draw(count) -> (tensor, event the consumer stream must wait for)."""
        return _GpuEpochSampler(self.device, num_items, random_state, total)

    # ---- evaluation on the item shards (mrr_score, precision_recall_score, predict) ----
    def bloom_item_rows(self, W_full, ids, seeds):
        """Item vectors of the global ids ``ids`` from the whole hashed table: the lookup
        ``BloomEmbedding.forward`` does (the sum of each id's hashed rows, padding id 0)."""
        return ops.embedding(W_full, ids, seeds, 0)

    def shard_scores(self, users, user_bias, items, item_bias):
        """(len(users), len(items)) scores with the arithmetic of evaluation._score_block: the GEMM,
        then += user bias, then += item bias."""
        out = users @ items.t()                             # plain library GEMM (cuBLAS)
        out += user_bias.reshape(-1, 1)
        out += item_bias.reshape(1, -1)
        return out

    def pair_scores(self, users, user_bias, items, item_bias, u_idx, i_idx):
        """scores[n] = <users[u_idx[n]], items[i_idx[n]]> + user_bias[u_idx[n]] + item_bias[i_idx[n]]:
        the kernel BilinearNet.forward runs on plain tables."""
        return ops.mf_scores(users, items, user_bias.reshape(-1, 1), item_bias.reshape(-1, 1), u_idx, i_idx)

    def rank_counts(self, scores, col_offset, row_ptr, targets, target_scores):
        """(3, n_targets) int32: slb_rank_counts' gt, eq and eq_before of every target over the block's
        columns, the global items [col_offset, col_offset + scores.shape[1]).  ``row_ptr`` and
        ``targets`` are host arrays in global item ids, ``target_scores`` the targets' full-row scores."""
        dev = target_scores.device
        scores = scores.contiguous()
        rp = torch.from_numpy(np.ascontiguousarray(row_ptr, dtype=np.int64)).to(dev)
        tg = torch.from_numpy(np.ascontiguousarray(targets, dtype=np.int64)).to(dev)
        n = tg.numel()
        out = torch.empty((3, n), dtype=torch.int32, device=dev)
        _lib.check(_lib.load().slb_rank_counts(ops._ptr(scores), scores.shape[0], scores.shape[1], col_offset,
                                               ops._ptr(rp), ops._ptr(tg), ops._ptr(target_scores.contiguous()), n,
                                               ops._ptr(out[0]), ops._ptr(out[1]), ops._ptr(out[2]), ops._stream()),
                   'rank_counts')
        return out

    # ---- sequence evaluation on the item shards (sequence scorers, predict) ----
    def seq_representation(self, E_cache, seqs_idx, cnn, lstm, mixture):
        """(n, S+1, width) causal representations of the sequences ``seqs_idx`` (ids remapped onto
        the row cache ``E_cache``, cache row 0 the padding row): ops.seq_representation, the kernels
        ``user_representation`` runs on a plain table.  width is D, or 2MD with ``mixture``."""
        return ops.seq_representation(E_cache, seqs_idx, cnn, lstm=lstm, mixture=mixture)

    def seq_dot_scores(self, final, items, item_bias):
        """(len(final), len(items)) scores of the dot head with the arithmetic of
        evaluation._score_sequences: the GEMM, then += item bias (no user bias)."""
        out = final @ items.t()                             # plain library GEMM (cuBLAS)
        out += item_bias.reshape(1, -1)
        return out

    def mixture_scores(self, final, items, item_bias):
        """(n, len(items)) scores of MixtureLSTMNet's mixture-of-tastes head for the final
        representations ``final`` (n, 2M, D): one slb_mixture_scores launch over the given rows."""
        n, two_m, dim = final.shape
        final, items, item_bias = final.contiguous(), items.contiguous(), item_bias.reshape(-1).contiguous()
        out = torch.empty((n, items.shape[0]), dtype=torch.float32, device=final.device)
        _lib.check(_lib.load().slb_mixture_scores(ops._ptr(final), n, two_m // 2, dim, ops._ptr(items),
                                                  ops._ptr(item_bias), items.shape[0], ops._ptr(out), ops._stream()),
                   'mixture_scores')
        return out

    def shard_mask_targets(self, scores, col_offset, excluded, row_ptr, targets):
        """slb_shard_mask_targets: writes -FLOAT_MAX, in place, over the excluded ids (device (n, L)
        int64, or None) inside the contiguous block's columns [col_offset, col_offset +
        scores.shape[1]) and returns the targets' scores (0 for a target outside the block).
        ``row_ptr`` and ``targets`` are host arrays in global item ids."""
        dev = scores.device
        rp = torch.from_numpy(np.ascontiguousarray(row_ptr, dtype=np.int64)).to(dev)
        tg = torch.from_numpy(np.ascontiguousarray(targets, dtype=np.int64)).to(dev)
        out = torch.empty(tg.numel(), dtype=torch.float32, device=dev)
        ex = None if excluded is None else excluded.contiguous()
        _lib.check(_lib.load().slb_shard_mask_targets(ops._ptr(scores), scores.shape[0], scores.shape[1], col_offset,
                                                      ops._ptr(ex), 0 if ex is None else ex.shape[1], ops._ptr(rp),
                                                      ops._ptr(tg), ops._ptr(out), ops._stream()),
                   'shard_mask_targets')
        return out

    def seq_local_step(self, E_cache, bias_cache, n_cache, seqs_idx, negs_idx, loss, cnn, norm_count,
                       lstm=None, mixture=None, n_neg=1):
        """Fused sequence step on the row cache (ids already remapped onto it; cache
        row 0 is the padding row).  Returns (loss share, dE_cache, dbias_cache, dconv_w, dconv_b,
        dlstm, dmix); ``lstm`` / ``mixture`` / ``n_neg`` as ops.seq_train_step takes them."""
        out = ops.seq_train_step(E_cache, bias_cache.reshape(-1, 1), seqs_idx, negs_idx, loss, n_neg, cnn,
                                 norm_count=norm_count, lstm=lstm, mixture=mixture)
        return (out['loss'], out['dE'][:n_cache], out['dbias'].reshape(-1)[:n_cache],
                out['dconv_w'], out['dconv_b'], out['dlstm'], out['dmix'])


_CHUNK_VALUES = 24 << 20        # negatives per sampler chunk: within the one-round reach of the jump table


class _GpuEpochSampler(object):
    def __init__(self, device, num_items, random_state, total):
        from spotlight_b200 import rng
        from spotlight_b200.factorization.implicit import _side_stream
        self.dev, self.num_items = torch.device(device), int(num_items)
        self.side = _side_stream(self.dev)
        self.out = torch.empty(total, dtype=torch.int64, device=self.dev)
        self.side.wait_stream(torch.cuda.current_stream(self.dev))
        with torch.cuda.stream(self.side):
            rng.reserve(self.num_items, total, self.dev)     # scratch sized once, before the first draw
            self.stream = rng.DeviceStream(random_state, self.dev)
        self.done = 0

    def draw(self, count):
        lo, self.done = self.done, self.done + count
        with torch.cuda.stream(self.side):
            self.stream.draw(self.num_items, count, out=self.out[lo:self.done])
            ev = torch.cuda.Event()
            ev.record(self.side)
        return self.out[lo:self.done], ev

    def finish(self):
        with torch.cuda.stream(self.side):
            self.stream.finish()
        self.out.record_stream(torch.cuda.current_stream(self.dev))


class _HostEpochSampler(object):
    """Backend-agnostic fallback: one synchronous draw per request (CPU / gloo tests)."""

    def __init__(self, backend, num_items, random_state):
        self.be, self.num_items, self.rs = backend, num_items, random_state

    def draw(self, count):
        return self.be.sample(self.num_items, count, self.rs), None

    def finish(self):
        pass


def adagrad_dense_(W, state, grad, lr, eps):
    """torch.optim.Adagrad update (lr_decay 0) on a small shard; rows with zero
    gradient are unchanged, so this equals the row-wise update of touched rows."""
    state.addcmul_(grad, grad)
    W.addcdiv_(grad, state.sqrt().add_(eps), value=-lr)


class ShardState(object):
    """This rank's parameter shards and their optimizer state.

    ``optimizer_func``: None (row-wise Adagrad at ``lr``, ``eps``), ``optim.fused_adagrad`` without
    weight decay (Adagrad with its ``lr``, ``eps``) or ``optim.fused_adam``; it is called on
    :meth:`params`.  Under ``fused_adam``, ``opt`` is that ``FusedAdam``: the user shard and its bias
    (``bu2``, the (rows, 1) view of ``bu``) and the item shard and its bias (``bi2``) are its two
    lazily updated table pairs, with moments ``mWu``, ``vWu``, ``mbu``, ``vbu`` / ``mWi``, ``vWi``,
    ``mbi``, ``vbi`` and the step each row is current for, ``last_u`` / ``last``.  A rank that owns no
    users registers the item pair only."""

    def __init__(self, plan, rank, dim, device, lr=0.05, eps=1e-10, init=None, optimizer_func=None):
        ulo, uhi = plan.user_range(rank)
        ilo, ihi = plan.item_range(rank)
        self.ulo, self.uhi, self.ilo, self.ihi = ulo, uhi, ilo, ihi
        self.lr, self.eps = float(lr), float(eps)
        dev = torch.device(device)
        rows = plan.ichunk              # item shards are padded to the common chunk: the whole-shard
        #                                 exchange (all-gather / reduce-scatter) runs on them directly;
        #                                 rows past ihi - ilo stay zero and are never addressed
        self.Wi = torch.zeros((rows, dim), device=dev)
        self.bi = torch.zeros(rows, device=dev)
        if init is not None:            # slices of full tables (tests / checkpoints)
            Wu, Wi, bu, bi = init
            self.Wu = Wu[ulo:uhi].clone().to(dev)
            self.Wi[:ihi - ilo] = Wi[ilo:ihi].to(dev)
            self.bu = bu[ulo:uhi].reshape(-1).clone().to(dev)
            self.bi[:ihi - ilo] = bi[ilo:ihi].reshape(-1).to(dev)
        else:
            self.Wu = torch.randn((uhi - ulo, dim), device=dev) / dim
            self.Wi[:ihi - ilo] = torch.randn((ihi - ilo, dim), device=dev) / dim
            self.bu = torch.zeros(uhi - ulo, device=dev)
        self.bu2, self.bi2 = self.bu.reshape(-1, 1), self.bi.reshape(-1, 1)
        self.opt = None
        state = torch.zeros_like                    # Adagrad's accumulators
        if optimizer_func is not None:
            from spotlight_b200.optim import FusedAdagrad, FusedAdam
            opt = optimizer_func(self.params())
            if isinstance(opt, FusedAdam):
                self.opt = opt
                self.mWi, self.vWi, self.last = opt.fused_states(self.Wi)
                self.mbi, self.vbi, _ = opt.fused_states(self.bi2)
                if self.Wu.shape[0]:
                    self.mWu, self.vWu, self.last_u = opt.fused_states(self.Wu)
                    self.mbu, self.vbu, _ = opt.fused_states(self.bu2)
                else:                               # no users here: nothing to step or flush
                    self.mWu, self.vWu = torch.zeros_like(self.Wu), torch.zeros_like(self.Wu)
                    self.mbu, self.vbu = torch.zeros_like(self.bu2), torch.zeros_like(self.bu2)
                    self.last_u = torch.zeros(0, dtype=torch.int32, device=dev)
                state = lambda p: None              # noqa: E731
            elif isinstance(opt, FusedAdagrad) and opt.fused_hparams()['weight_decay'] == 0:
                hp = opt.fused_hparams()
                self.lr, self.eps = hp['lr'], hp['eps']
            else:
                # fused_adagrad's weight decay moves the rows a minibatch updates, which the owners
                # do not see as the single-process step does
                raise ValueError('the sharded factorization model trains with optimizer_func=None (row-wise '
                                 'Adagrad at learning_rate), optim.fused_adagrad without weight decay or '
                                 'optim.fused_adam; got %s' % type(opt).__name__)
        self.sWu, self.sWi = state(self.Wu), state(self.Wi)
        self.sbu, self.sbi = state(self.bu), state(self.bi)

    def params(self):
        """The table pairs (user shard, its bias as a (rows, 1) view, item shard, its bias) -- the user
        pair only when this rank owns users."""
        return ([self.Wu, self.bu2] if self.Wu.shape[0] else []) + [self.Wi, self.bi2]


def _global_loss(loss_share, group):
    """The global minibatch loss: the sum of the ranks' shares (one scalar all-reduce)."""
    total = loss_share.detach().clone().reshape(1)
    dist.all_reduce(total, group=group)
    return total.reshape(())


def _reduce_scatter(x, chunk, rank, group):
    """This rank's ``chunk`` rows of the sum over ranks of ``x`` (``world * chunk`` rows)."""
    out = x.new_empty((chunk,) + tuple(x.shape[1:]))
    try:
        dist.reduce_scatter_tensor(out, x, group=group)
    except (RuntimeError, NotImplementedError):          # gloo: sum everywhere, keep our slice
        y = x.clone()
        dist.all_reduce(y, group=group)
        out.copy_(y[rank * chunk:(rank + 1) * chunk])
    return out


class _RowExchange(object):
    """The per-row item exchange of the MF and sequence steps (module docstring): the distinct
    item ids of a rank's batch are bucketed by owner and requested with an all-to-all, the owners
    gather the rows and biases from their shard and send them back, and after the local step the
    gradient rows travel home the same way.  The owner-side update is the caller's."""

    def __init__(self, plan, state, rank, backend, group=None, cache_capacity=None):
        self.plan, self.st, self.rank, self.backend, self.group = plan, state, rank, backend, group
        self.cache_capacity = cache_capacity
        self.stats = {'rows_requested': 0, 'bytes_a2a': 0}

    def _a2a(self, send, send_counts, recv_counts):
        out = send.new_empty((sum(recv_counts),) + tuple(send.shape[1:]))
        dist.all_to_all_single(out, send.contiguous(), output_split_sizes=list(recv_counts),
                               input_split_sizes=list(send_counts), group=self.group)
        self.stats['bytes_a2a'] += out.numel() * out.element_size()
        return out

    def _fetch_rows(self, ids, before_gather=None):
        """Distinct item rows of ``ids`` from their owners: returns (cache_rows, cache_bias,
        inverse, n_cache, route) with ``ids[k]`` living in cache row ``inverse[k]``.
        ``before_gather(local_req)`` runs at the owner on the shard rows its peers requested,
        before it gathers them."""
        plan, st, P = self.plan, self.st, self.plan.world
        dev = ids.device
        if ids.numel():
            uniq, inverse, bounds = self.backend.unique_bucket(ids, plan.num_items, plan.ichunk, P)
        else:                               # nothing of this minibatch lives here: serve peers only
            uniq, inverse, bounds = ids, ids, [0] * (P + 1)
        send_counts = [bounds[p + 1] - bounds[p] for p in range(P)]
        sc = torch.tensor(send_counts, dtype=torch.int64, device=dev)
        rc = torch.empty(P, dtype=torch.int64, device=dev)
        dist.all_to_all_single(rc, sc, group=self.group)
        recv_counts = rc.tolist()
        req = self._a2a(uniq, send_counts, recv_counts)
        local_req = req - st.ilo
        if before_gather is not None:
            before_gather(local_req)
        rows, bias = self.backend.gather(st.Wi, st.bi, local_req)
        n_cache = uniq.numel()
        # fixed capacity (a function of the batch shape only) so the fused step's workspace is reused
        cap = self.cache_capacity or min(ids.numel(), plan.num_items)
        cache_rows = self._a2a(rows, recv_counts, send_counts)
        cache_bias = self._a2a(bias, recv_counts, send_counts)
        if cap > n_cache:
            full = cache_rows.new_zeros((cap, cache_rows.shape[1]))
            full[:n_cache] = cache_rows
            fb = cache_bias.new_zeros(cap)
            fb[:n_cache] = cache_bias
            cache_rows, cache_bias = full, fb
        self.stats['rows_requested'] += n_cache
        return cache_rows, cache_bias, inverse, n_cache, (send_counts, recv_counts, local_req)

    def _return_grads(self, route, g_rows, g_bias):
        """Item gradient rows go home: returns (local_req, g_recv, gb_recv), the shard rows this
        owner served and the gradient rows and biases its peers sent for them, in rank order."""
        send_counts, recv_counts, local_req = route
        g_recv = self._a2a(g_rows.contiguous(), send_counts, recv_counts)
        gb_recv = self._a2a(g_bias.contiguous(), send_counts, recv_counts)
        return local_req, g_recv, gb_recv


class ShardedMF(_RowExchange):
    """BPR/hinge/pointwise matrix factorisation with range-sharded rows."""

    def _dense_exchange_pays(self, local_batch):
        """When a rank's 2*B item draws cover most of the table anyway, the
        per-row routing (bucketing + 3 variable all-to-alls + two host syncs) moves
        as many bytes as shipping whole shards; then all-gather / reduce-scatter of
        the shards is the cheaper exchange."""
        return 2 * local_batch >= self.plan.num_items

    def step(self, users, items, negs, loss, global_batch, exchange='auto', n_neg=1):
        """One training step on this rank's share of the global minibatch.

        ``exchange``: 'a2a' (per-row routing), 'dense' (whole-shard all-gather /
        reduce-scatter) or 'auto'.  ``negs`` holds ``B * n_neg`` ids (adaptive hinge:
        the flat ``randint`` block of the reference, implicit.py:266-275; its user
        pairing ``users[f // n]`` is local because every user of this rank's batch
        is owned by this rank).
        """
        if loss == 'adaptive_hinge' or n_neg != 1:
            # the reference's pairing spans the global minibatch: see step_adaptive
            raise ValueError('adaptive hinge needs the minibatch positions: use step_adaptive')
        if exchange == 'dense' or (exchange == 'auto' and
                                   self._dense_exchange_pays(global_batch // self.plan.world)):
            return self.step_dense(users, items, negs, loss, global_batch, n_neg)
        return self.step_a2a(users, items, negs, loss, global_batch, n_neg)

    def step_dense(self, users, items, negs, loss, global_batch, n_neg=1):
        """Whole-shard exchange: all-gather the item shards, fused local step on the
        full (transient) item table with raw ids, reduce-scatter the dense item
        gradient back to its owners.  No bucketing, no host synchronisation."""
        plan, st, P = self.plan, self.st, self.plan.world
        chunk, D = plan.ichunk, st.Wi.shape[1]
        dev = users.device
        adam, kw = st.opt is not None, {}
        if adam:                            # lazy-exact Adam: every rank gathers every row, current through t - 1
            t = st.opt.steps_taken + 1
            kw = {'t': t}
            self.backend.owner_adam_catch_up_shard(st, t - 1)
        pad_W, pad_b = st.Wi, st.bi          # shards are stored padded to the common chunk
        full_W = st.Wi.new_empty((P * chunk, D))
        full_b = st.bi.new_empty(P * chunk)
        dist.all_gather_into_tensor(full_W, pad_W, group=self.group)
        dist.all_gather_into_tensor(full_b, pad_b, group=self.group)
        self.stats['bytes_a2a'] += (full_W.numel() + full_b.numel()) * 4
        self.stats['rows_requested'] += P * chunk
        if users.numel():
            loss_share, g_rows, g_bias = self.backend.local_step(
                st, full_W, full_b, P * chunk, users - st.ulo, items, negs, loss, global_batch, n_neg, **kw)
        else:                               # none of this minibatch's users live here
            loss_share, g_rows, g_bias = full_b.new_zeros(()), torch.zeros_like(full_W), torch.zeros_like(full_b)
        g_shard = _reduce_scatter(g_rows.contiguous(), chunk, self.rank, self.group)
        gb_shard = _reduce_scatter(g_bias.contiguous(), chunk, self.rank, self.group)
        self.stats['bytes_a2a'] += (g_rows.numel() + g_bias.numel()) * 4
        n = st.Wi.shape[0]
        if adam:                            # dense Adam step t on the whole shard, then count it
            self.backend.adam_dense(st, False, g_shard[:n], gb_shard[:n], t)
            st.opt.advance(1)
        else:
            adagrad_dense_(st.Wi, st.sWi, g_shard[:n], st.lr, st.eps)
            adagrad_dense_(st.bi, st.sbi, gb_shard[:n], st.lr, st.eps)
        return _global_loss(loss_share, self.group)

    def step_a2a(self, users, items, negs, loss, global_batch, n_neg=1):
        """Per-row routing (the north-star exchange).

        ``users`` must all be owned by this rank (global ids).  Returns the
        *global* mean loss as a 0-dim tensor (identical on every rank).
        """
        st = self.st
        B = users.numel()
        catch_up, kw = self._adam_hooks()
        cache_rows, cache_bias, inverse, n_cache, route = self._fetch_rows(torch.cat([items, negs]), catch_up)
        # fused local step (user rows updated in place)
        if B:
            loss_share, g_rows, g_bias = self.backend.local_step(
                st, cache_rows, cache_bias, n_cache, users - st.ulo, inverse[:B], inverse[B:], loss,
                global_batch, n_neg, **kw)
        else:
            loss_share, g_rows, g_bias = st.bi.new_zeros(()), cache_rows[:0], cache_bias[:0]
        self._owner_step(self._return_grads(route, g_rows, g_bias), kw)
        return _global_loss(loss_share, self.group)

    def _adam_hooks(self):
        """(before_gather, local-step keywords) of this step: under lazy-exact Adam the owner catches
        the requested rows up through t - 1 before it gathers them, and the step is t."""
        st = self.st
        if st.opt is None:
            return None, {}
        t = st.opt.steps_taken + 1
        return (lambda local_req: self.backend.owner_adam_catch_up(st, local_req, t)), {'t': t}    # noqa: E731

    def _owner_step(self, returned, kw):
        """The owner's update of the rows its peers returned gradients for: Adagrad, or Adam step t,
        which every rank then counts (also a rank without members, so t stays equal everywhere)."""
        if not kw:
            self.backend.owner_update(self.st, *returned)
            return
        self.backend.owner_adam_update(self.st, *returned, kw['t'])
        self.st.opt.advance(1)

    def step_adaptive(self, users, items, negs_block, bpos, batch_users, n_neg):
        """Adaptive hinge on a sharded minibatch, with the reference's pairing.

        The reference scores flat negative f of a minibatch with ``users[f // n]`` and
        reads the result as element ``(k, b) = (f // B, f % B)`` of the ``(n, B)`` matrix
        whose column maxima enter the hinge (implicit.py:266-275, losses.py:127-166).  So
        a negative is *scored* where interaction ``f // n`` lives and *consumed* where
        interaction ``f % B`` lives.  Each rank scores the n-blocks of its own members
        (``negs_block[j*n:(j+1)*n]`` are flats ``bpos[j]*n ..``), the 4-byte scores travel
        to the owners of their columns, the loss and the arg-max gradients are formed
        there, and the gradients travel back the same way.  Rows never move for this:
        only the usual item-row exchange around it.
        """
        plan, st, P = self.plan, self.st, self.plan.world
        be = self.backend
        m, Bg, n = users.numel(), batch_users.numel(), int(n_neg)
        dev = users.device
        catch_up, kw = self._adam_hooks()
        cache_rows, cache_bias, inverse, n_cache, route = self._fetch_rows(torch.cat([items, negs_block]), catch_up)
        ul = users - st.ulo
        ul_rep = ul.repeat_interleave(n)
        # scores of this rank's members and of their n-blocks
        if m:
            if kw:
                # the user rows scored current through t - 1 (the others catch up in adam_dense below)
                be.user_adam_catch_up(st, ul, kw['t'])
            pos = be.scores(st, cache_rows, cache_bias, ul, inverse[:m])
            neg = be.scores(st, cache_rows, cache_bias, ul_rep, inverse[m:])
        else:
            pos = st.bi.new_zeros(0)
            neg = st.bi.new_zeros(0)
        # flats -> owners of their columns
        flat = (bpos.repeat_interleave(n) * n + torch.arange(n, device=dev).repeat(m)) if m else bpos
        dest = torch.div(batch_users[flat % Bg], plan.uchunk, rounding_mode='floor') if m else bpos
        order = torch.argsort(dest, stable=True)
        send_counts = torch.bincount(dest, minlength=P)
        recv_counts_t = torch.empty_like(send_counts)
        dist.all_to_all_single(recv_counts_t, send_counts, group=self.group)
        sc, rc = send_counts.tolist(), recv_counts_t.tolist()
        f_recv = self._a2a(flat[order], sc, rc)
        s_recv = self._a2a(neg[order], sc, rc)
        # the (n, m) matrix of this rank's columns, loss, gradients
        if m:
            lookup = torch.full((Bg,), -1, dtype=torch.int64, device=dev)
            lookup[bpos] = torch.arange(m, device=dev)
            slot = torch.div(f_recv, Bg, rounding_mode='floor') * m + lookup[f_recv % Bg]
            negmat = s_recv.new_empty(n * m)
            negmat[slot] = s_recv
            loss_mean, gp, gn = be.adaptive_loss(pos, negmat.reshape(n, m))
            # hinge gradients are exactly -/+ 1/B_global wherever they are non-zero: emit that
            # value itself (not (1/m) * (m/B), which rounds differently per rank), so that
            # +g and -g meeting on one row cancel exactly as they do in one process
            inv = float(np.float32(1.0) / np.float32(Bg))
            loss_share = loss_mean * (m / float(Bg))
            gp = torch.where(gp != 0, -inv, 0.0).to(torch.float32)
            g_back = torch.where(gn.reshape(-1)[slot] != 0, inv, 0.0).to(torch.float32)
        else:
            loss_share, gp, g_back = st.bi.new_zeros(()), pos, s_recv
        g_sorted = self._a2a(g_back, rc, sc)
        # backward of the scores, with the gradient each score earned at its consumer
        if m:
            g_neg = torch.empty_like(g_sorted)
            g_neg[order] = g_sorted
            dWu, dcache, dbu, dbcache = be.scores_backward(
                st, cache_rows, torch.cat([gp, g_neg]), torch.cat([ul, ul_rep]), inverse)
            if kw:                          # dense Adam step t on the user shard
                be.adam_dense(st, True, dWu, dbu, kw['t'])
            else:
                adagrad_dense_(st.Wu, st.sWu, dWu, st.lr, st.eps)
                adagrad_dense_(st.bu, st.sbu, dbu.reshape(-1), st.lr, st.eps)
            g_rows, g_bias = dcache[:n_cache], dbcache.reshape(-1)[:n_cache]
        else:
            g_rows, g_bias = cache_rows[:0], cache_bias[:0]
        self._owner_step(self._return_grads(route, g_rows, g_bias), kw)
        return _global_loss(loss_share, self.group)


class SeqShardState(object):
    """Item-embedding / item-bias shards, the replicated representation parameters and their
    optimizer state.  ``convs``: list of (weight (D,D,k,1), bias (D,)) of CNNNet; ``lstm``:
    dict(w_ih, w_hh, b_ih, b_hh) of LSTMNet / MixtureLSTMNet; ``mixture``: dict(num_mixtures,
    w (2MD, D, 1), b (2MD,)), MixtureLSTMNet's projection (the forms ops.seq_train_step takes).

    ``optimizer_func``: None (row-wise Adagrad at ``lr``, ``eps``), ``optim.fused_adagrad`` without
    weight decay (Adagrad with its ``lr``, ``eps``) or ``optim.fused_adam``; it is called on
    :meth:`params`.  Under ``fused_adam``, ``opt`` is that ``FusedAdam``: the item shard and its bias
    (``bi2``, the (rows, 1) view of ``bi``) are its lazily updated table pair, with ``mWi``, ``vWi``,
    ``last``, ``mbi``, ``vbi`` their moments and the step each row is current for; the replicated
    parameters take its dense ``step()``."""

    def __init__(self, plan, rank, dim, device, lr=0.05, eps=1e-10, init=None, convs=None, lstm=None,
                 mixture=None, optimizer_func=None):
        ilo, ihi = plan.item_range(rank)
        self.ilo, self.ihi = ilo, ihi
        self.lr, self.eps = float(lr), float(eps)
        dev = torch.device(device)
        if init is not None:
            E, bias = init
            self.Wi = E[ilo:ihi].clone().to(dev)
            self.bi = bias[ilo:ihi].reshape(-1).clone().to(dev)
        else:
            self.Wi = torch.randn((ihi - ilo, dim), device=dev) / dim
            self.bi = torch.zeros(ihi - ilo, device=dev)
            if ilo == 0:
                self.Wi[0] = 0                      # padding row (PADDING_IDX = 0)
        self.bi2 = self.bi.reshape(-1, 1)
        # conv weights are replicated: list of (weight (D,D,k,1), bias (D,)) tensors
        self.convs = [(w.clone().to(dev), b.clone().to(dev)) for w, b in (convs or [])]
        self.lstm = None if lstm is None else {k: lstm[k].detach().clone().to(dev).contiguous()
                                               for k in ('w_ih', 'w_hh', 'b_ih', 'b_hh')}
        self.mixture = None
        if mixture is not None:
            self.mixture = dict(num_mixtures=int(mixture['num_mixtures']),
                                w=mixture['w'].detach().clone().to(dev).contiguous(),
                                b=mixture['b'].detach().clone().to(dev).contiguous())
        self.opt = None
        state = torch.zeros_like                    # Adagrad's accumulators
        if optimizer_func is not None:
            from spotlight_b200.optim import FusedAdagrad, FusedAdam
            opt = optimizer_func(self.params())
            if isinstance(opt, FusedAdam):
                self.opt = opt
                self.mWi, self.vWi, self.last = opt.fused_states(self.Wi)
                self.mbi, self.vbi, _ = opt.fused_states(self.bi2)
                state = lambda p: None              # noqa: E731
            elif isinstance(opt, FusedAdagrad) and opt.fused_hparams()['weight_decay'] == 0:
                hp = opt.fused_hparams()
                self.lr, self.eps = hp['lr'], hp['eps']
            else:
                # fused_adagrad's weight decay moves the rows a minibatch updates, which the owners
                # do not see as the single-process step does
                raise ValueError('the sharded sequence model trains with optimizer_func=None (row-wise Adagrad at '
                                 'learning_rate), optim.fused_adagrad without weight decay or optim.fused_adam; '
                                 'got %s' % type(opt).__name__)
        self.sWi, self.sbi = state(self.Wi), state(self.bi)
        self.srep = [state(p) for p in self.params()[2:]]

    def params(self):
        """The item shard, its bias as a (rows, 1) view and the replicated parameters, in a fixed
        order."""
        out = [self.Wi, self.bi2] + [p for wb in self.convs for p in wb]
        if self.lstm is not None:
            out += [self.lstm[k] for k in ('w_ih', 'w_hh', 'b_ih', 'b_hh')]
        if self.mixture is not None:
            out += [self.mixture[k] for k in ('w', 'b')]
        return out

    def replicated(self):
        """(parameter, Adagrad state) pairs of the replicated parameters, in a fixed order (state
        None under Adam)."""
        return list(zip(self.params()[2:], self.srep))


class ShardedSeq(_RowExchange):
    """PoolNet / CNNNet / LSTMNet / MixtureLSTMNet training step with range-sharded item rows
    (SURVEY §8e, config 5).

    Sequences are data-parallel (each rank owns whole sequences); every item row a
    rank's batch touches -- as input, target or negative -- is fetched once per step by
    the same bucket -> all-to-all -> gather -> all-to-all exchange as the MF step, the
    fused sequence kernels run on the row cache, and the per-row gradients return to
    their owners.  The loss is normalised by the *global* number of unmasked positions
    (one scalar all-reduce up front); conv, LSTM and projection weights are replicated
    (``state``) and their gradients all-reduced.  ``n_neg`` negatives per position
    (adaptive hinge): ``negs`` holds ``n_neg * B`` rows, row ``q * B + b`` for sequence ``b``.
    """

    def __init__(self, plan, state, rank, backend, cnn=None, group=None, cache_capacity=None, n_neg=1):
        _RowExchange.__init__(self, plan, state, rank, backend, group, cache_capacity)
        self.cnn = cnn                      # dict(kernel_width, dilation, nonlinearity, residual) or None
        self.n_neg = int(n_neg)

    def step(self, seqs, negs, loss):
        st = self.st
        B, S = seqs.shape
        # global mask count first (device scalar; no host sync)
        norm = (seqs != 0).sum().to(torch.int32).reshape(1)
        dist.all_reduce(norm, group=self.group)
        # distinct ids, with the padding id forced in so that it maps to cache row 0
        ids = torch.cat([seqs.reshape(-1), negs.reshape(-1), seqs.new_zeros(1)])
        adam = st.opt is not None
        catch_up = None
        if adam:                            # lazy-exact Adam: the requested rows current through t - 1
            t = st.opt.steps_taken + 1
            catch_up = lambda local_req: self.backend.owner_adam_catch_up(st, local_req, t)    # noqa: E731
        cache_rows, cache_bias, inverse, n_cache, route = self._fetch_rows(ids, catch_up)
        n, nn = B * S, self.n_neg
        if B:
            cnn = None
            if self.cnn is not None:
                cnn = dict(self.cnn, weights=[w for w, _ in st.convs], biases=[b for _, b in st.convs])
            # lstm / mixture / n_neg are passed only when used, so a backend that knows only
            # PoolNet / CNNNet keeps working for those nets
            extra = {}
            if st.lstm is not None:
                extra['lstm'] = st.lstm
            if st.mixture is not None:
                extra['mixture'] = st.mixture
            if nn != 1:
                extra['n_neg'] = nn
            out = self.backend.seq_local_step(
                cache_rows, cache_bias, n_cache, inverse[:n].reshape(B, S),
                inverse[n:n + nn * n].reshape(nn * B, S), loss, cnn, norm, **extra)
            loss_share, g_rows, g_bias = out[:3]
            grads = [g for pair in zip(out[3], out[4]) for g in pair]
            dlstm, dmix = (out[5], out[6]) if len(out) > 5 else (None, None)
            if st.lstm is not None:
                grads += [dlstm[k] for k in ('w_ih', 'w_hh', 'b_ih', 'b_hh')]
            if st.mixture is not None:
                grads += [dmix[k] for k in ('w', 'b')]
        else:                               # no sequence of this minibatch here: serve peers, join the reductions
            loss_share = cache_bias.new_zeros(())
            g_rows, g_bias = cache_rows.new_zeros((n_cache, cache_rows.shape[1])), cache_bias.new_zeros(n_cache)
            grads = [torch.zeros_like(p) for p, _ in st.replicated()]
        returned = self._return_grads(route, g_rows, g_bias)
        if adam:
            # step t on the received rows, then FusedAdam.step() takes step t on the replicated
            # parameters (the only ones carrying a .grad) and counts it, as the single-GPU route does
            self.backend.owner_adam_update(st, *returned, t)
            for (p, _), g in zip(st.replicated(), grads):
                dist.all_reduce(g, group=self.group)
                p.grad = g.reshape(p.shape)
            st.opt.step()
            for p, _ in st.replicated():
                p.grad = None
        else:
            self.backend.owner_update(st, *returned)
            for (p, s), g in zip(st.replicated(), grads):
                dist.all_reduce(g, group=self.group)
                self.backend.adagrad_dense(p, s, g.reshape(p.shape), st.lr, st.eps)
        return _global_loss(loss_share, self.group)


def _rank_slice(n, rank, world):
    """[lo, hi) of this rank's near-equal contiguous share of n rows (the first n % world ranks
    take one more)."""
    base, extra = divmod(n, world)
    lo = rank * base + min(rank, extra)
    return lo, lo + base + (1 if rank < extra else 0)


class ShardedImplicitSequenceModel(object):
    """``ImplicitSequenceModel.fit`` on N GPUs (one process per GPU, one instance per rank), with
    the *single-process* semantics of the reference loop (sequence/implicit.py:193-264):

    * the constructor draws the torch seed from ``random_state`` and builds the net on the CPU as
      the single-process model does, so a string ``representation`` starts from the same weights;
      each rank then keeps only its item range of the embedding table and bias, the
      representation's own parameters (conv, LSTM, projection) are replicated;
    * per epoch one shuffle of the sequence rows (applied cumulatively) and one
      ``sample_items(num_items, (n_seq * n_neg, S))`` draw, from the one global stream that every
      rank advances identically;
    * minibatch k is rows ``[k*B, (k+1)*B)``; each rank trains a near-equal contiguous slice of it
      and the loss and gradients are those of the whole minibatch (:class:`ShardedSeq`);
    * ``epoch_loss`` is the mean of the global minibatch losses.

    Every rank is handed the same ``SequenceInteractions``.  Optimizer (``optimizer_func``):

    * ``None``: row-wise Adagrad at ``learning_rate`` on the item rows
      (``spotlight_b200.optim.fused_adagrad``'s update) and Adagrad on the replicated parameters;
      ``fused_adagrad(lr, eps)`` without weight decay is the same with its hyper-parameters;
    * ``fused_adam(lr, betas, eps, weight_decay)``: row-wise lazy-exact Adam on the item rows at
      their owners and Adam on the replicated parameters at the same step count -- the trajectory
      of ``ImplicitSequenceModel(optimizer_func=fused_adam(...))``, i.e. dense ``torch.optim.Adam``
      on every parameter, weight decay included, up to fp32 rounding.  ``fit()`` brings every
      row current before it returns, and repeated calls resume the step count and the moments;
    * anything else raises ``ValueError``.

    Nets: PoolNet, CNNNet, LSTMNet, MixtureLSTMNet on a plain
    ``ScaledEmbedding(padding_idx=0)`` within the fused step's limits (``net.fusable()``); any
    other net raises ``ValueError``.

    Evaluation, on the shards: ``evaluation.sequence_mrr_score`` and
    ``evaluation.sequence_precision_recall_score`` take this model, and :meth:`predict` scores items
    for one sequence; all three are collective (every rank calls them with the same arguments and
    gets the whole result) and gather no table whole.
    """

    def __init__(self, num_items, rank, world, device, loss='pointwise', representation='pooling',
                 embedding_dim=32, n_iter=10, batch_size=256, learning_rate=1e-2, random_state=None,
                 num_negative_samples=5, group=None, backend=None, optimizer_func=None):
        from spotlight_b200.sequence.representations import CNNNet, LSTMNet, MixtureLSTMNet, PoolNet
        from spotlight_b200.torch_utils import set_seed
        assert loss in ('pointwise', 'bpr', 'hinge', 'adaptive_hinge')
        self._loss, self._n_iter, self._batch_size = loss, int(n_iter), int(batch_size)
        self._n_neg = int(num_negative_samples) if loss == 'adaptive_hinge' else 1
        self._num_items = int(num_items)
        self._random_state = random_state or np.random.RandomState()
        self.rank, self.world, self.device = rank, world, torch.device(device)
        self.backend = backend or GpuBackend(device)
        # the single-process model seeds torch from its stream at construction (implicit.py:124)
        # and builds the net from that seed (_initialize)
        set_seed(self._random_state.randint(-10 ** 8, 10 ** 8), cuda=self.device.type == 'cuda')
        builders = {'pooling': PoolNet, 'cnn': CNNNet, 'lstm': LSTMNet, 'mixture': MixtureLSTMNet}
        if isinstance(representation, str):
            net = builders[representation](self._num_items, embedding_dim)
        else:
            net = representation
        if not (isinstance(net, (PoolNet, CNNNet, LSTMNet, MixtureLSTMNet)) and net.fusable()):
            raise ValueError('ShardedImplicitSequenceModel trains PoolNet, CNNNet, LSTMNet and MixtureLSTMNet '
                             'on a plain ScaledEmbedding(padding_idx=0) within the fused step\'s limits '
                             '(embedding_dim % 4 == 0); got %s' % type(net).__name__)
        if net.item_embeddings.num_embeddings != self._num_items:
            raise ValueError('representation has %d item rows, the model %d'
                             % (net.item_embeddings.num_embeddings, self._num_items))
        self._net = net
        D = net.embedding_dim
        self.plan = ShardPlan(1, self._num_items, world)
        cnn = net._cnn_spec()
        self.state = SeqShardState(
            self.plan, rank, D, self.device, lr=learning_rate,
            init=(net.item_embeddings.weight.detach(), net.item_biases.weight.detach()),
            convs=[(w.detach(), b.detach()) for w, b in zip(cnn['weights'], cnn['biases'])] if cnn else None,
            lstm=net._lstm_spec(), mixture=net._mixture_spec(), optimizer_func=optimizer_func)
        spec = None if cnn is None else {k: cnn[k] for k in ('kernel_width', 'dilation', 'nonlinearity', 'residual')}
        self.seq = ShardedSeq(self.plan, self.state, rank, self.backend, cnn=spec, group=group, n_neg=self._n_neg)
        self.epoch_losses = []

    def fit(self, interactions, verbose=False):
        """Fit the model; repeated calls resume (implicit.py:193-264)."""
        sequences = interactions.sequences
        if torch.is_tensor(sequences):
            seqs = sequences.to(self.device, torch.int64).contiguous()
        else:
            seqs = self.backend.to_device(np.asarray(sequences).astype(np.int64))
        n_seq = seqs.shape[0]
        if n_seq and int(seqs.max()) >= self._num_items:
            raise ValueError('Maximum item id greater than number of items in model.')
        B, nn, S = self._batch_size, self._n_neg, seqs.shape[1]
        for epoch in range(self._n_iter):
            order = self.backend.shuffled_order(n_seq, self._random_state)
            seqs = seqs.index_select(0, order.to(seqs.device))
            del order
            negatives = self.backend.sample(self._num_items, (n_seq * nn, S), self._random_state)
            epoch_loss = torch.zeros((), dtype=torch.float64, device=seqs.device)
            nbatch = 0
            for lo in range(0, n_seq, B):
                m = min(B, n_seq - lo)
                a, c = _rank_slice(m, self.rank, self.world)
                # the minibatch's negatives are rows q*m + b of its (nn*m, S) block; ours are b in [a, c)
                block = negatives[lo * nn:(lo + m) * nn].reshape(nn, m, S)
                mine = block[:, a:c].reshape(nn * (c - a), S)
                loss = self.seq.step(seqs[lo + a:lo + c], mine, self._loss)
                epoch_loss += loss.detach().double()
                nbatch += 1
            epoch_loss = float(epoch_loss.item()) / max(nbatch, 1)
            self.epoch_losses.append(epoch_loss)
            if verbose and self.rank == 0:
                print('Epoch {}: loss {}'.format(epoch, epoch_loss))
            if np.isnan(epoch_loss) or epoch_loss == 0.0:
                raise ValueError('Degenerate epoch loss: {}'.format(epoch_loss))
        if self.state.opt is not None:
            self.backend.owner_adam_flush(self.state)       # lazy-exact Adam: every row current
        return self

    def gathered_net(self):
        """Collective: the representation module on this rank's device with the full trained item
        table and bias (all-gathered from the shards) and the replicated parameters.  The sequence
        scorers and :meth:`predict` score the sharded model itself, without gathering it."""
        st, plan = self.state, self.plan
        full = []
        for shard in (st.Wi, st.bi.reshape(-1, 1)):
            pad = shard.new_zeros((plan.ichunk,) + tuple(shard.shape[1:]))
            pad[:shard.shape[0]] = shard
            parts = [torch.empty_like(pad) for _ in range(self.world)]
            dist.all_gather(parts, pad, group=self.seq.group)
            full.append(torch.cat(parts)[:self._num_items])
        net = self._net.to(self.device)
        with torch.no_grad():
            net.item_embeddings.weight.copy_(full[0])
            net.item_biases.weight.copy_(full[1])
            mine = []
            for layer in (getattr(net, 'cnn_layers', None) or []):
                mine += [layer.weight, layer.bias]
            if st.lstm is not None:
                mine += [net.lstm.weight_ih_l0, net.lstm.weight_hh_l0, net.lstm.bias_ih_l0, net.lstm.bias_hh_l0]
            if st.mixture is not None:
                mine += [net.projection.weight, net.projection.bias]
            for prm, (val, _) in zip(mine, st.replicated()):
                prm.copy_(val.reshape(prm.shape))
        return net

    # ------------------------------------------------------------------ evaluation
    def _final_representations(self, seqs):
        """Collective: the final representations of the block ``seqs`` (host int64 (n, S), the same on
        every rank), in block order on every rank: (n, D), or (n, 2M, D) for MixtureLSTMNet (block j
        of the projection's channels j*D + d, the layout evaluation._mixture_block scores).

        Rank r builds those of its contiguous slice ``_rank_slice(n, r, world)`` on a row cache of the
        slice's distinct items, fetched from their owners as a training step fetches them, with id 0
        forced in so that padding lands on cache row 0 (PoolNet's mask reads the row's values).  A rank
        with an empty slice still serves its peers' rows.  The slices, padded to ceil(n / world) rows,
        are all-gathered."""
        st, be, seq, world = self.state, self.backend, self.seq, self.world
        n, S = seqs.shape
        a, c = _rank_slice(n, self.rank, world)
        mine = be.to_device(np.ascontiguousarray(seqs[a:c], dtype=np.int64))
        cache_rows, _, inverse, _, _ = seq._fetch_rows(torch.cat([mine.reshape(-1), mine.new_zeros(1)]))
        D = st.Wi.shape[1]
        width = D if st.mixture is None else 2 * st.mixture['num_mixtures'] * D
        per = -(-n // world)
        part = cache_rows.new_zeros((per, width))
        if c > a:
            cnn = None
            if seq.cnn is not None:
                cnn = dict(seq.cnn, weights=[w for w, _ in st.convs], biases=[b for _, b in st.convs])
            rep = be.seq_representation(cache_rows, inverse[:(c - a) * S].reshape(c - a, S), cnn, st.lstm,
                                        st.mixture)
            part[:c - a] = rep[:, -1]
        full = part.new_empty((world * per, width))
        dist.all_gather_into_tensor(full, part, group=seq.group)
        sizes = [hi - lo for lo, hi in (_rank_slice(n, r, world) for r in range(world))]
        final = full[be.to_device(np.concatenate([r * per + np.arange(m) for r, m in enumerate(sizes)]))]
        return final if st.mixture is None else final.reshape(n, -1, D)

    def _shard_scores(self, final, items, item_bias):
        """(n, len(items)) scores of the final representations against the item rows given, with
        the single-GPU scorer's arithmetic: the dot head's GEMM then += bias, or the mixture head."""
        if self.state.mixture is None:
            return self.backend.seq_dot_scores(final, items, item_bias)
        return self.backend.mixture_scores(final, items, item_bias)

    def _eval_blocks(self, inputs, targets, exclude_preceding, sequence_block):
        """Collective: yields (first row, (3, n * k) int64 counts gt, eq, eq_before over all items) for
        every block of ``sequence_block`` input sequences; ``targets`` (n_seq, k) holds each
        sequence's targets in global item ids.

        Per block: the final representations are built on the slices and all-gathered, each rank
        scores them against its item range, pushes the block's input items inside the range to the
        bottom (``exclude_preceding``) and reads the targets it owns (slb_shard_mask_targets); the
        targets' scores, then the rank counts of every range, are all-reduced.  A rank that owns no
        items scores nothing and joins every collective."""
        st, be, group = self.state, self.backend, self.seq.group
        k = targets.shape[1]
        for lo in range(0, len(inputs), sequence_block):
            blk = np.ascontiguousarray(inputs[lo:lo + sequence_block], dtype=np.int64)
            n = len(blk)
            final = self._final_representations(blk)
            if st.ihi == st.ilo:
                scores = final.new_empty((n, 0))
            else:
                if st.mixture is None:
                    # the operand layout evaluation._score_sequences hands its GEMM (the last step of an
                    # (n, S+1, D) representation), so that the library takes the same algorithm for it
                    steps = final.new_empty((n, blk.shape[1] + 1, final.shape[1]))
                    steps[:, -1] = final
                    final = steps[:, -1]
                scores = self._shard_scores(final, st.Wi, st.bi)
            tg = targets[lo:lo + n].reshape(-1)
            row_ptr = np.arange(n + 1) * k
            target_scores = be.shard_mask_targets(scores, st.ilo, be.to_device(blk) if exclude_preceding else None,
                                                  row_ptr, tg)
            dist.all_reduce(target_scores, group=group)
            counts = be.rank_counts(scores, st.ilo, row_ptr, tg, target_scores)
            dist.all_reduce(counts, group=group)
            yield lo, counts.cpu().numpy().astype(np.int64)

    def predict(self, sequences, item_ids=None):
        """Collective: scores of ``item_ids`` (all items when None) as the next item of one sequence,
        a flat NumPy array on every rank -- ``ImplicitSequenceModel.predict``'s arguments and result.
        Every rank calls it with the same arguments.  Each rank scores the requested items it owns,
        from their rows gathered contiguously, against the sequence's final representation; the
        zero-filled outputs are all-reduced.  ``fit()`` leaves every row current, so the model can be
        scored as it stands."""
        st, be = self.state, self.backend
        seqs = np.atleast_2d(sequences).astype(np.int64).reshape(1, -1)
        items = (np.arange(self._num_items, dtype=np.int64) if item_ids is None
                 else np.asarray(item_ids).astype(np.int64).reshape(-1))
        for ids in (items, seqs):                   # every rank raises before any collective
            if ids.size and ids.max() >= self._num_items:
                raise ValueError('Maximum item id greater than number of items in model.')
            if ids.size and ids.min() < 0:
                raise ValueError('Item ids must not be negative.')
        final = self._final_representations(seqs)
        own = np.nonzero((items >= st.ilo) & (items < st.ihi))[0]
        out = torch.zeros(len(items), dtype=torch.float32, device=st.Wi.device)
        if len(own):
            rows, bias = be.gather(st.Wi, st.bi, be.to_device(items[own] - st.ilo))
            out[be.to_device(own)] = self._shard_scores(final, rows, bias)[0]
        dist.all_reduce(out, group=self.seq.group)
        return out.cpu().numpy()


class ShardedImplicitFactorizationModel(object):
    """``ImplicitFactorizationModel.fit`` on N GPUs (one process per GPU), with the
    *single-process* semantics of the reference loop (factorization/implicit.py:184-252):

    * one global ``RandomState`` stream, advanced identically on every rank: the epoch
      permutation (``shuffle``) and the negatives (``sample_items`` once per minibatch) are
      the reference's, bit for bit;
    * minibatch k is ``shuffled[k*B:(k+1)*B]`` of the *global* data set; each rank trains
      the members whose user it owns and the loss / gradients are those of the whole
      minibatch (:class:`ShardedMF`);
    * ``epoch_loss`` is the mean of the global minibatch losses.

    Every rank is handed the same ``Interactions`` (the global shuffle needs all of it);
    parameters and optimizer state are sharded, never replicated.  All four losses; adaptive
    hinge keeps the reference's global negative pairing (:meth:`ShardedMF.step_adaptive`).
    Optimizer (``optimizer_func``):

    * ``None``: row-wise Adagrad at ``learning_rate`` (``spotlight_b200.optim.fused_adagrad``'s
      update); ``fused_adagrad(lr, eps)`` without weight decay is the same with its hyper-parameters;
    * ``fused_adam(lr, betas, eps, weight_decay)``: row-wise lazy-exact Adam on the user shard and on
      the item shard at its owners -- the trajectory of
      ``ImplicitFactorizationModel(optimizer_func=fused_adam(...))``, i.e. dense ``torch.optim.Adam``
      on all four tables, weight decay included, up to fp32 rounding.  ``fit()`` brings every row
      current before it returns, and repeated calls resume the step count and the moments;
    * anything else raises ``ValueError``.

    ``representation``: a ``BilinearNet`` with a plain user layer and a ``BloomEmbedding(padding_idx=0)``
    item layer (BASELINE config 4) trains from that net's weights on :class:`ShardedBloomMF`: user
    shards, the hashed table sharded by row range and exchanged whole, the item bias replicated.
    Pointwise, bpr and hinge, under either optimizer above; ``exchange`` 'auto' or 'dense' (the
    hashed table always travels whole).  Anything else raises ``ValueError``.  :meth:`gathered_net`
    returns the trained net of either kind.

    Evaluation, on the shards: ``evaluation.mrr_score`` and ``evaluation.precision_recall_score`` take
    this model, and :meth:`predict` scores pairs; all three are collective (every rank calls them with
    the same arguments and gets the whole result) and gather no table whole.  They score the model as
    it stands: ``fit()`` leaves every lazily updated row current, so nothing is needed between the two.
    """

    def __init__(self, num_users, num_items, rank, world, device, backend=None, loss='bpr',
                 embedding_dim=32, n_iter=10, batch_size=256, learning_rate=0.05, random_state=None,
                 exchange='auto', init=None, group=None, num_negative_samples=5, optimizer_func=None,
                 representation=None):
        assert loss in ('pointwise', 'bpr', 'hinge', 'adaptive_hinge')
        self._n_neg = int(num_negative_samples) if loss == 'adaptive_hinge' else 1
        self._loss, self._n_iter, self._batch_size = loss, int(n_iter), int(batch_size)
        self._num_users, self._num_items = int(num_users), int(num_items)
        self._random_state = random_state or np.random.RandomState()
        self._exchange = exchange
        self.rank, self.world, self.device = rank, world, torch.device(device)
        self.plan = ShardPlan(num_users, num_items, world)
        self.backend = backend or GpuBackend(device)
        self._net = None
        if representation is not None:
            self._check_bloom_net(representation)
        # the reference seeds torch from the model stream at construction (implicit.py:114);
        # the draw is kept so that the stream position matches the single-process model
        seed = int(self._random_state.randint(-10 ** 8, 10 ** 8))
        if representation is not None:
            net = self._net = representation
            layer = net.item_embeddings
            init = [t.detach() for t in (net.user_embeddings.weight, layer.embeddings.weight,
                                         net.user_biases.weight, net.item_biases.weight)]
            self.state = BloomShardState(self.plan, rank, net.embedding_dim, device, self._num_items,
                                         layer.compressed_num_embeddings, layer.num_hash_functions,
                                         lr=learning_rate, init=init, optimizer_func=optimizer_func)
            self.mf = ShardedBloomMF(self.plan, self.state, rank, self.backend, group=group)
        else:
            if init is None:
                torch.manual_seed(seed + 7919 * rank)
            self.state = ShardState(self.plan, rank, embedding_dim, device, lr=learning_rate, init=init,
                                    optimizer_func=optimizer_func)
            self.mf = ShardedMF(self.plan, self.state, rank, self.backend, group=group)
        self.epoch_losses = []

    def _check_bloom_net(self, net):
        """ValueError unless ``net`` is a BilinearNet that :class:`ShardedBloomMF` trains as given."""
        from spotlight_b200.factorization.representations import BilinearNet
        from spotlight_b200.layers import BloomEmbedding, ScaledEmbedding
        if self._loss == 'adaptive_hinge':
            raise ValueError('the sharded Bloom model trains pointwise, bpr and hinge; adaptive hinge needs the '
                             'per-row exchange')
        if self._exchange == 'a2a':
            raise ValueError("the sharded Bloom model exchanges the hashed table whole: exchange='auto' or 'dense'")
        if not isinstance(net, BilinearNet):
            raise ValueError('representation must be a BilinearNet; got %s' % type(net).__name__)
        ul, il = net.user_embeddings, net.item_embeddings
        if type(ul) is not ScaledEmbedding or ul.padding_idx is not None:
            raise ValueError('the sharded Bloom model takes a plain user layer (ScaledEmbedding without padding); '
                             'got %s' % type(ul).__name__)
        if type(il) is not BloomEmbedding or getattr(il, '_bag', False) or il.padding_idx != 0:
            raise ValueError('the sharded Bloom model takes a BloomEmbedding(bag=False, padding_idx=0) item layer; '
                             'got %r' % (il,))
        if ul.sparse or il.embeddings.sparse or net.user_biases.sparse or net.item_biases.sparse:
            raise ValueError('the sharded Bloom model takes dense gradients: build the net with sparse=False')
        if net.embedding_dim % 4:
            raise ValueError('the sharded Bloom model needs embedding_dim % 4 == 0')
        if ul.num_embeddings != self._num_users or net.user_biases.num_embeddings != self._num_users:
            raise ValueError('representation has %d user rows, the model %d' % (ul.num_embeddings, self._num_users))
        if il.num_embeddings != self._num_items or net.item_biases.num_embeddings != self._num_items:
            raise ValueError('representation has %d item ids, the model %d' % (il.num_embeddings, self._num_items))

    def gathered_net(self):
        """Collective: the trained ``BilinearNet`` on this rank's device, its tables all-gathered from
        the shards (a Bloom model: the representation it was built from, its replicated item bias as
        it is).  ``mrr_score``, ``precision_recall_score`` and :meth:`predict` score the sharded model
        itself, on its shards, without gathering it."""
        from spotlight_b200.factorization.representations import BilinearNet
        st, plan = self.state, self.plan

        def gather(shard, chunk, n):
            pad = shard.new_zeros((chunk,) + tuple(shard.shape[1:]))
            pad[:shard.shape[0]] = shard
            parts = [torch.empty_like(pad) for _ in range(self.world)]
            dist.all_gather(parts, pad, group=self.mf.group)
            return torch.cat(parts)[:n]

        Wu = gather(st.Wu, plan.uchunk, self._num_users)
        bu = gather(st.bu.reshape(-1, 1), plan.uchunk, self._num_users)
        if self._net is not None:
            net = self._net.to(self.device)
            Wi, Wi_dst = gather(st.Wi, st.mchunk, st.M), net.item_embeddings.embeddings.weight
            bi = st.bi.reshape(-1, 1)
        else:
            net = BilinearNet(self._num_users, self._num_items, st.Wu.shape[1]).to(self.device)
            Wi, Wi_dst = gather(st.Wi, plan.ichunk, self._num_items), net.item_embeddings.weight
            bi = gather(st.bi.reshape(-1, 1), plan.ichunk, self._num_items)
        with torch.no_grad():
            net.user_embeddings.weight.copy_(Wu)
            net.user_biases.weight.copy_(bu)
            Wi_dst.copy_(Wi)
            net.item_biases.weight.copy_(bi)
        return net

    # ------------------------------------------------------------------ evaluation
    def _hashed_table(self):
        """Collective: the whole hashed item table (M rows) of a Bloom model, all-gathered."""
        st = self.state
        W_full = st.Wi.new_empty((self.world * st.mchunk, st.Wi.shape[1]))
        dist.all_gather_into_tensor(W_full, st.Wi, group=self.mf.group)
        return W_full[:st.M]

    def _user_rows(self, users):
        """Collective: (rows (n, D), biases (n,)) of the global user ids ``users`` (host int64) on every
        rank.  Each owner writes its users into a zero buffer and one all-reduce sums it: every
        element has a single non-zero contributor, so the sum is exact."""
        st, be = self.state, self.backend
        D = st.Wu.shape[1]
        buf = torch.zeros((len(users), D + 1), dtype=torch.float32, device=st.Wu.device)
        mine = np.nonzero((users >= st.ulo) & (users < st.uhi))[0]
        if len(mine):
            rows, local = be.to_device(mine.astype(np.int64)), be.to_device((users[mine] - st.ulo).astype(np.int64))
            buf[rows, :D] = st.Wu[local]
            buf[rows, D] = st.bu[local]
        dist.all_reduce(buf, group=self.mf.group)
        return buf[:, :D].contiguous(), buf[:, D].contiguous()

    def _check_ids(self, users, items):
        """ValueError, raised on every rank before any collective (all ranks hold the same ids)."""
        if len(users) and (users.min() < 0 or users.max() >= self._num_users):
            raise ValueError('User ids must lie in [0, %d), the model\'s number of users.' % self._num_users)
        if len(items) and (items.min() < 0 or items.max() >= self._num_items):
            raise ValueError('Item ids must lie in [0, %d), the model\'s number of items.' % self._num_items)

    def _eval_blocks(self, test, train, user_block):
        """Collective: yields (first output row, CSR test rows of the block, (3, n_targets) int64 counts
        gt, eq, eq_before over all items) for every block of ``user_block`` users with test items.

        Per block: the user rows are all-reduced, each rank scores them against its item range, pushes
        the train items inside the range to the bottom, and the targets' scores (written by their
        owners) and then the rank counts of every range are all-reduced."""
        be, group = self.backend, self.mf.group
        test = test.tocsr()
        train = train.tocsr() if train is not None else None
        for m in (test, train):
            if m is not None:
                self._check_ids(np.nonzero(np.diff(m.indptr))[0], m.indices)
        ilo, ihi = self.plan.item_range(self.rank)
        st = self.state
        if self._net is None:
            items, item_bias = st.Wi[:ihi - ilo], st.bi[:ihi - ilo]
        else:
            ids = torch.arange(ilo, ihi, dtype=torch.int64, device=st.Wi.device)
            items, item_bias = be.bloom_item_rows(self._hashed_table(), ids, st.item_seeds), st.bi[ilo:ihi]
        users = np.nonzero(np.diff(test.indptr))[0]
        for lo in range(0, len(users), user_block):
            blk = users[lo:lo + user_block]
            u, ub = self._user_rows(blk)
            scores = be.shard_scores(u, ub, items, item_bias)
            if train is not None:
                tr = train[blk]
                rows, cols = np.repeat(np.arange(len(blk)), np.diff(tr.indptr)), tr.indices
                keep = (cols >= ilo) & (cols < ihi)
                if keep.any():
                    scores[be.to_device(rows[keep].astype(np.int64)),
                           be.to_device((cols[keep] - ilo).astype(np.int64))] = -float(np.finfo(np.float32).max)
            te = test[blk]
            rows, targets = np.repeat(np.arange(len(blk)), np.diff(te.indptr)), te.indices.astype(np.int64)
            target_scores = torch.zeros(len(targets), dtype=torch.float32, device=scores.device)
            own = np.nonzero((targets >= ilo) & (targets < ihi))[0]
            if len(own):
                target_scores[be.to_device(own.astype(np.int64))] = scores[be.to_device(rows[own].astype(np.int64)),
                                                                           be.to_device(targets[own] - ilo)]
            dist.all_reduce(target_scores, group=group)
            counts = be.rank_counts(scores, ilo, te.indptr, targets, target_scores)
            dist.all_reduce(counts, group=group)
            yield lo, te, counts.cpu().numpy().astype(np.int64)

    def predict(self, user_ids, item_ids=None):
        """Collective: scores of (user, item) pairs, or of one user against ``item_ids`` (all items when
        None), as a NumPy array on every rank -- ``ImplicitFactorizationModel.predict``'s arguments and
        result.  Every rank calls it with the same ids.  Each pair is scored by the rank that owns its
        item, from the all-reduced user rows; the zero-filled outputs are all-reduced.  The model must
        be current: ``fit()`` brings every lazily updated row up to date before it returns."""
        from spotlight_b200.factorization._components import _predict_process_ids
        st, be = self.state, self.backend
        users, items = _predict_process_ids(user_ids, item_ids, self._num_items, False)
        users, items = users.numpy(), items.numpy()
        self._check_ids(users, items)
        uniq, inverse = np.unique(users, return_inverse=True)
        U, ub = self._user_rows(uniq)
        W_full = None if self._net is None else self._hashed_table()
        ilo, ihi = self.plan.item_range(self.rank)
        own = np.nonzero((items >= ilo) & (items < ihi))[0]
        out = torch.zeros(len(items), dtype=torch.float32, device=st.Wu.device)
        if len(own):
            u_idx = be.to_device(inverse.reshape(-1)[own].astype(np.int64))
            if W_full is None:
                s = be.pair_scores(U, ub, st.Wi, st.bi, u_idx, be.to_device(items[own] - ilo))
            else:
                ids = be.to_device(items[own])
                s = be.pair_scores(U, ub, be.bloom_item_rows(W_full, ids, st.item_seeds), st.bi[ids], u_idx,
                                   torch.arange(len(own), dtype=torch.int64, device=out.device))
            out[be.to_device(own.astype(np.int64))] = s
        dist.all_reduce(out, group=self.mf.group)
        return out.cpu().numpy()

    def fit(self, interactions, verbose=False):
        be = self.backend
        n = len(interactions.user_ids)
        if hasattr(be, 'upload_sharded'):
            users_dev = be.upload_sharded(interactions.user_ids, self.rank, self.world, self.mf.group)
            items_dev = be.upload_sharded(interactions.item_ids, self.rank, self.world, self.mf.group)
        else:
            users_dev = be.to_device(interactions.user_ids)
            items_dev = be.to_device(interactions.item_ids)
        if users_dev.dtype != items_dev.dtype:
            users_dev, items_dev = users_dev.long(), items_dev.long()
        if n:
            umax, imax = torch.stack([users_dev.max(), items_dev.max()]).tolist()      # one sync
            if umax >= self._num_users:
                raise ValueError('Maximum user id greater than number of users in model.')
            if imax >= self._num_items:
                raise ValueError('Maximum item id greater than number of items in model.')
        for epoch in range(self._n_iter):
            order = be.shuffled_order(n, self._random_state)
            u, i = be.permute(order, users_dev, items_dev)
            del order
            epoch_loss = self._run_epoch_device(u, i)
            del u, i
            self.epoch_losses.append(epoch_loss)
            if verbose and self.rank == 0:
                print('Epoch {}: loss {}'.format(epoch, epoch_loss))
            if np.isnan(epoch_loss) or epoch_loss == 0.0:
                raise ValueError('Degenerate epoch loss: {}'.format(epoch_loss))
        if self.state.opt is not None:
            be.owner_adam_flush(self.state)                 # lazy-exact Adam: every row current
        return self

    def _run_epoch_device(self, u, i):
        """One epoch over the (already shuffled) global ids ``u`` / ``i``, held identically on
        every rank's device: global negative stream (chunked, on a side stream where the
        backend has one), owner partition, and the sharded steps of this rank's members.
        Returns the epoch loss (mean of the global minibatch losses, implicit.py:240,245)."""
        plan, be, B, nn = self.plan, self.backend, self._batch_size, self._n_neg
        n = u.numel()
        if n == 0:
            return 0.0
        # this rank's members of every minibatch, in minibatch order (no dependence on negatives)
        ulo, uhi = plan.user_range(self.rank)
        mine = torch.nonzero((u >= ulo) & (u < uhi)).reshape(-1)
        edges = torch.arange(0, n + B, B, device=mine.device).clamp_(max=n)
        bounds = torch.searchsorted(mine, edges).tolist()                   # the epoch's one sync
        bloom = self._net is not None
        dense = not bloom and (self._exchange == 'dense' or (self._exchange == 'auto' and
                                                             self.mf._dense_exchange_pays(B // plan.world)))
        if dense and nn == 1 and isinstance(be, GpuBackend) and self.state.opt is None:
            return self._epoch_dense_gpu(u, i, mine, bounds)
        mu, mi = u[mine], i[mine]
        bpos = mine % B
        sampler = (be.epoch_sampler(self._num_items, self._random_state, n * nn)
                   if hasattr(be, 'epoch_sampler') else _HostEpochSampler(be, self._num_items, self._random_state))
        nsteps = len(bounds) - 1
        losses = []
        k, cur = 0, max(1, _CHUNK_VALUES // (B * nn))
        while k < nsteps:
            # one draw per chunk of global minibatches; a minibatch draws len(batch) * n values at
            # once (implicit.py:256-259, 266-275): the n-block of the member at epoch position p
            # is negs[n*p : n*p + n]
            hi_k = min(k + cur, nsteps)
            lo_e, hi_e = k * B, min(hi_k * B, n)
            negs, ev = sampler.draw((hi_e - lo_e) * nn)
            if ev is not None:
                torch.cuda.current_stream(u.device).wait_event(ev)
            negs = negs.reshape(hi_e - lo_e, nn)
            for kk in range(k, hi_k):
                sl = slice(bounds[kk], bounds[kk + 1])
                mn = negs[mine[sl] - lo_e].reshape(-1)
                if bloom:
                    losses.append(self.mf.step(mu[sl], mi[sl], mn, self._loss, min(B, n - kk * B)))
                elif self._loss == 'adaptive_hinge':
                    losses.append(self.mf.step_adaptive(mu[sl], mi[sl], mn, bpos[sl], u[kk * B:(kk + 1) * B], nn))
                else:
                    losses.append(self.mf.step(mu[sl], mi[sl], mn, self._loss, min(B, n - kk * B),
                                               self._exchange))
            k = hi_k
        sampler.finish()
        return float(torch.stack(losses).mean()) if losses else 0.0

    # ------------------------------------------------------------------ fast path
    def _buffers(self, key, make):
        cache = self.__dict__.setdefault('_buf_cache', {})
        if key not in cache:
            cache[key] = make()
        return cache[key]

    def _epoch_dense_gpu(self, u, i, mine, bounds):
        """Whole-shard exchange epoch on the product kernels with nothing but launches on the
        host side of the loop: per global minibatch k

          plan stream   gather this rank's members (one kernel), integer plan of the local step
                        (csrc/mf_v2.cuh) -- one step ahead, double buffered
          main stream   all-gather of the item shards -> mf_user_kernel (user rows updated in
                        place) -> mf_item_kernel (dense item gradient) -> reduce-scatter ->
                        Adagrad on the owned shard

        The global negative stream is drawn on the sampler's side stream in chunks; the loss
        shares are all-reduced once per epoch.  Same arithmetic as ShardedMF.step_dense.
        """
        from spotlight_b200.factorization.implicit import _plan_stream
        lib = _lib.load()
        be, st, plan, P = self.backend, self.state, self.plan, self.plan.world
        dev = u.device
        B, n = self._batch_size, u.numel()
        nsteps = len(bounds) - 1
        D, chunk = st.Wi.shape[1], plan.ichunk
        main, pstream = torch.cuda.current_stream(dev), _plan_stream(dev)
        loss_kind = _lib.LOSS_KIND[self._loss]
        maxm = max(1, max(bounds[k + 1] - bounds[k] for k in range(nsteps)))
        cap = 1 << (maxm - 1).bit_length()                    # capacity bucket: buffers are reused across epochs
        buf = self._buffers(('dense', cap), lambda: dict(
            full_W=torch.empty((P * chunk, D), device=dev), full_b=torch.empty(P * chunk, device=dev),
            dW=torch.empty((P * chunk, D), device=dev), db=torch.empty(P * chunk, device=dev),
            gW=torch.empty((chunk, D), device=dev), gb=torch.empty(chunk, device=dev),
            ids=[[torch.empty(cap, dtype=torch.int64, device=dev) for _ in range(3)] for _ in range(2)]))
        U_sh, I_all = st.Wu.shape[0], P * chunk
        fws = ops.workspace('mfv2_%d_%d_%d' % (U_sh, I_all, D), lib.slb_mf_fused_workspace_bytes(cap, U_sh, I_all, D), dev)
        ws = ops.workspace('mf%d_%d' % (U_sh, I_all), lib.slb_mf_step_workspace_bytes(cap, 1, loss_kind, U_sh, I_all), dev)
        assert fws.numel() > 0, 'planned step unavailable for dim %d' % D
        losses = torch.zeros(nsteps, dtype=torch.float32, device=dev)
        sampler = be.epoch_sampler(self._num_items, self._random_state, n)
        # The whole stream is enqueued up front in chunks as large as one jump round reaches
        # (~24 M values): a chunk costs one latency-bound jump round + one fill round whatever its
        # size, and that generator slows down several-fold when it shares SMs with the training
        # kernels -- so as much as possible is drawn before the first step (measured at N = 4: the
        # 1, 2, 4, 8-batch doubling schedule stalled 20 steps for 27 ms in total).
        waits = []                                             # (first step, event) per chunk of negatives
        per = max(1, _CHUNK_VALUES // B)
        k = 0
        while k < nsteps:
            hi_k = min(k + per, nsteps)
            _, ev = sampler.draw(min(hi_k * B, n) - k * B)
            waits.append((k, ev))
            k = hi_k
        negs_all = sampler.out
        plan_ev = [torch.cuda.Event(), torch.cuda.Event()]
        done_ev = [torch.cuda.Event(), torch.cuda.Event()]
        pstream.wait_stream(main)                              # ids, tables and buffers are ready
        args = [None, None]
        next_wait = [0]

        def make_args(k):
            # runs on the plan stream: the workspaces are the main stream's, which the step reads
            ul, it, ng = buf['ids'][k & 1]
            a = _users_only_args(st, buf['full_W'], buf['full_b'], ul, it, ng, loss_kind, 1, buf['dW'], buf['db'],
                                 min(B, n - k * B), batch=bounds[k + 1] - bounds[k], workspaces=(ws, fws))
            a.loss_out = losses[k:k + 1].data_ptr()
            return a

        def prep(k):
            slot = k & 1
            m = bounds[k + 1] - bounds[k]
            with torch.cuda.stream(pstream):
                while next_wait[0] < len(waits) and waits[next_wait[0]][0] <= k:
                    pstream.wait_event(waits[next_wait[0]][1])
                    next_wait[0] += 1
                if k >= 2:
                    pstream.wait_event(done_ev[slot])          # the slot's ids / plan are free again
                args[slot] = make_args(k)
                if m:
                    ul, it, ng = buf['ids'][slot]
                    _lib.check(lib.slb_shard_gather_batch(
                        ops._ptr(mine[bounds[k]:]), m, ops._ptr(u), ops._ptr(i), ops._ptr(negs_all), 0, 1,
                        st.ulo, ops._ptr(ul), ops._ptr(it), ops._ptr(ng), ops._stream()), 'shard_gather_batch')
                    _lib.check(lib.slb_mf_train_step_phases(ctypes.byref(args[slot]), 1 | (slot << 8),
                                                            ops._stream()), 'plan')
                plan_ev[slot].record(pstream)

        prep(0)
        for k in range(nsteps):
            if k + 1 < nsteps:
                prep(k + 1)
            slot = k & 1
            m = bounds[k + 1] - bounds[k]
            dist.all_gather_into_tensor(buf['full_W'], st.Wi, group=self.mf.group)
            dist.all_gather_into_tensor(buf['full_b'], st.bi, group=self.mf.group)
            buf['dW'].zero_()
            buf['db'].zero_()
            main.wait_event(plan_ev[slot])
            if m:
                _lib.check(lib.slb_mf_train_step_phases(ctypes.byref(args[slot]), 6 | (slot << 8),
                                                        ops._stream()), 'step')
            done_ev[slot].record(main)
            dist.reduce_scatter_tensor(buf['gW'], buf['dW'], group=self.mf.group)
            dist.reduce_scatter_tensor(buf['gb'], buf['db'], group=self.mf.group)
            _lib.check(lib.slb_adagrad_dense(ops._ptr(st.Wi), ops._ptr(st.sWi), ops._ptr(buf['gW']), chunk * D,
                                             st.lr, st.eps, ops._stream()), 'adagrad')
            _lib.check(lib.slb_adagrad_dense(ops._ptr(st.bi), ops._ptr(st.sbi), ops._ptr(buf['gb']), chunk,
                                             st.lr, st.eps, ops._stream()), 'adagrad')
        # each step moved what ShardedMF.step_dense counts: the whole table there and its gradient back
        self.mf.stats['rows_requested'] += nsteps * P * chunk
        self.mf.stats['bytes_a2a'] += nsteps * 2 * (buf['full_W'].numel() + buf['full_b'].numel()) * 4
        pstream.wait_stream(main)                              # later plan-stream work follows this epoch
        dist.all_reduce(losses, group=self.mf.group)           # one reduction per epoch: global minibatch losses
        sampler.finish()
        host = losses.cpu().numpy().astype(np.float64)
        if ops.workspace_error_flag(ws):
            raise ValueError('ids out of range reached the device kernels')
        return float(host.mean()) if nsteps else 0.0


class BloomShardState(object):
    """Parameters of BilinearNet(plain users, BloomEmbedding items) on one rank: user rows / user
    bias sharded by user range, the hashed item table (M rows) sharded by row range and padded to
    the common chunk, the item bias (one float per raw item id) REPLICATED -- its forward lookup
    needs 2 values per interaction from arbitrary owners, which would cost a host-synchronised
    all-to-all per step for 4-byte payloads; its replicas are kept identical by applying the same
    all-gathered sparse updates on every rank.

    ``optimizer_func`` as :class:`ShardState`'s: None (row-wise Adagrad at ``lr``, ``eps``),
    ``optim.fused_adagrad`` without weight decay or ``optim.fused_adam``, called on :meth:`params`.
    Under ``fused_adam``, ``opt`` is that ``FusedAdam`` with three kinds of lazily updated table: the
    user shard and its bias (``bu2``, (rows, 1)) as a pair sharing ``last_u`` (registered only when
    this rank owns users), the hashed shard with its own ``last_i`` and the replicated item bias
    (``bi2``) with its own ``last_bi``; moments ``mWu``, ``vWu``, ``mbu``, ``vbu``, ``mWi``, ``vWi``,
    ``mbi``, ``vbi``."""

    def __init__(self, plan, rank, dim, device, num_ids, hashed_rows, num_hash, lr=0.05, eps=1e-10, init=None,
                 optimizer_func=None):
        from spotlight_b200.layers import SEEDS
        dev = torch.device(device)
        self.lr, self.eps = float(lr), float(eps)
        self.world = plan.world
        self.ulo, self.uhi = plan.user_range(rank)
        self.M, self.num_ids = int(hashed_rows), int(num_ids)
        self.mchunk = -(-self.M // plan.world)
        self.mlo = min(rank * self.mchunk, self.M)
        self.mhi = min(self.mlo + self.mchunk, self.M)
        self.item_seeds = [int(x) for x in SEEDS[:num_hash]]
        self.Wi = torch.zeros((self.mchunk, dim), device=dev)
        if init is not None:
            Wu, Wi, bu, bi = init
            self.Wu = Wu[self.ulo:self.uhi].clone().to(dev)
            self.bu = bu[self.ulo:self.uhi].reshape(-1).clone().to(dev)
            self.Wi[:self.mhi - self.mlo] = Wi[self.mlo:self.mhi].to(dev)
            self.bi = bi.reshape(-1).clone().to(dev)
        else:
            self.Wu = torch.randn((self.uhi - self.ulo, dim), device=dev) / dim
            self.bu = torch.zeros(self.uhi - self.ulo, device=dev)
            self.Wi[:self.mhi - self.mlo] = torch.randn((self.mhi - self.mlo, dim), device=dev) / dim
            if self.mlo == 0:
                self.Wi[0] = 0                      # padding row of the hashed table
            self.bi = torch.zeros(self.num_ids, device=dev)
        self.bu2, self.bi2 = self.bu.reshape(-1, 1), self.bi.reshape(-1, 1)
        self.opt = None
        state = torch.zeros_like                    # Adagrad's accumulators
        if optimizer_func is not None:
            from spotlight_b200.optim import FusedAdagrad, FusedAdam
            opt = optimizer_func(self.params())
            if isinstance(opt, FusedAdam):
                self.opt = opt
                self.mWi, self.vWi, self.last_i = opt.fused_states(self.Wi, own_last=True)
                self.mbi, self.vbi, self.last_bi = opt.fused_states(self.bi2, own_last=True)
                if self.Wu.shape[0]:
                    self.mWu, self.vWu, self.last_u = opt.fused_states(self.Wu)
                    self.mbu, self.vbu, _ = opt.fused_states(self.bu2)
                else:                               # no users here: nothing to step or flush
                    self.mWu, self.vWu = torch.zeros_like(self.Wu), torch.zeros_like(self.Wu)
                    self.mbu, self.vbu = torch.zeros_like(self.bu2), torch.zeros_like(self.bu2)
                    self.last_u = torch.zeros(0, dtype=torch.int32, device=dev)
                state = lambda p: None              # noqa: E731
            elif isinstance(opt, FusedAdagrad) and opt.fused_hparams()['weight_decay'] == 0:
                hp = opt.fused_hparams()
                self.lr, self.eps = hp['lr'], hp['eps']
            else:
                # fused_adagrad's weight decay moves the rows a minibatch updates, which the owners
                # do not see as the single-process step does
                raise ValueError('the sharded factorization model trains with optimizer_func=None (row-wise '
                                 'Adagrad at learning_rate), optim.fused_adagrad without weight decay or '
                                 'optim.fused_adam; got %s' % type(opt).__name__)
        self.sWu, self.sWi = state(self.Wu), state(self.Wi)
        self.sbu, self.sbi = state(self.bu), state(self.bi)

    def params(self):
        """The user shard and its bias as a (rows, 1) view (when this rank owns users), the hashed
        shard and the replicated item bias as a (num_ids, 1) view."""
        return ([self.Wu, self.bu2] if self.Wu.shape[0] else []) + [self.Wi, self.bi2]


class ShardedBloomMF(object):
    """Training step of the hashed-item model on N ranks (SURVEY section 8e, BASELINE config 4:
    BloomEmbedding 50 M items -> 1 M hashed rows, hinge / bpr / pointwise).

    Interactions are routed to the rank that owns their user (user gathers and updates local).
    The hashed table is range-sharded; a rank's minibatch references 2 * B * H hashed rows -- at
    config 4 sizes a large fraction of all M rows -- so the table travels whole: all-gather of the
    shards, the fused hashed step on the full table (in-register murmur3, layers.py:178-204) with
    the user rows and user biases updated in place (users-only mode, O(batch)), reduce-scatter of the
    dense table gradient to the owners, who step their whole shard.  The id-space item-bias
    gradients travel as (id, g) pairs: all-gather, then the same sparse update on every replica, in
    rank order.  Loss: one scalar all-reduce.

    Under lazy-exact Adam (``state.opt``) the step is t = ``steps_taken + 1`` on every rank, also on
    a rank without members in the minibatch: it contributes a zero gradient and no pairs, and steps
    its shard and the replica all the same.  The owners' dense step leaves every hashed row current
    through t, so the next all-gather needs no catch-up."""

    def __init__(self, plan, state, rank, backend, group=None, pair_capacity=None):
        self.plan, self.st, self.rank, self.backend, self.group = plan, state, rank, backend, group
        self.pair_capacity = pair_capacity
        self.stats = {'bytes_exchanged': 0}

    def step(self, users, items, negs, loss, global_batch):
        st, P, be = self.st, self.plan.world, self.backend
        dev = st.Wi.device
        D = st.Wi.shape[1]
        adam = st.opt is not None
        kw = {'t': st.opt.steps_taken + 1} if adam else {}
        W_full = st.Wi.new_empty((P * st.mchunk, D))
        dist.all_gather_into_tensor(W_full, st.Wi, group=self.group)
        m = users.numel()
        cap = self.pair_capacity or 2 * int(global_batch)
        ids_pad = torch.zeros(cap, dtype=torch.int64, device=dev)
        g_pad = torch.zeros(cap, dtype=torch.float32, device=dev)
        if m:
            loss_share, dWu, dWi, upairs, (ii, gi) = be.bloom_local_step(st, W_full[:st.M], users - st.ulo, items,
                                                                         negs, loss, global_batch, **kw)
            if dWu is not None:             # a backend that hands the user gradient out: Adagrad here
                be.adagrad_dense(st.Wu, st.sWu, dWu, st.lr, st.eps)
                be.bias_sparse_adagrad(upairs[0], upairs[1], st.bu, st.sbu, st.lr, st.eps)
            ids_pad[:ii.numel()] = ii
            g_pad[:gi.numel()] = gi
            if dWi.shape[0] == P * st.mchunk:
                dW_pad = dWi
            else:
                dW_pad = dWi.new_zeros((P * st.mchunk, D))
                dW_pad[:st.M] = dWi
        else:
            loss_share = st.bu.new_zeros(())
            dW_pad = st.Wi.new_zeros((P * st.mchunk, D))
        g_shard = _reduce_scatter(dW_pad, st.mchunk, self.rank, self.group)
        if adam:
            be.bloom_adam_dense(st, g_shard, kw['t'])
        else:
            be.adagrad_dense(st.Wi, st.sWi, g_shard, st.lr, st.eps)
        ids_all = torch.empty(P * cap, dtype=torch.int64, device=dev)
        g_all = torch.empty(P * cap, dtype=torch.float32, device=dev)
        dist.all_gather_into_tensor(ids_all, ids_pad, group=self.group)
        dist.all_gather_into_tensor(g_all, g_pad, group=self.group)
        if adam:
            # the zero padding pairs (id 0, g 0) take a real step for id 0: dense Adam steps every id
            # with a zero gradient too, so that step is exact
            be.bloom_bias_adam(st, ids_all, g_all, kw['t'])
            st.opt.advance(1)
        else:
            be.bias_sparse_adagrad(ids_all, g_all, st.bi, st.sbi, st.lr, st.eps)
        self.stats['bytes_exchanged'] += (W_full.numel() + dW_pad.numel()) * 4 + P * cap * 12
        return _global_loss(loss_share, self.group)


# ---------------------------------------------------------------- evaluation on the item shards

def _finalize_ranks(counts):
    """(average rank as float64 of its float32 value, stable position int64) from the all-reduced
    (3, n) counts gt, eq, eq_before: the float32 expression of rank_targets_kernel's rt_write
    (csrc/embed.cu), so that equal counts give slb_rank_targets' ranks bit for bit."""
    gt, eq, eq_before = counts
    avg = np.float32(1.0) + gt.astype(np.float32) + np.float32(0.5) * (eq - 1).astype(np.float32)
    return avg.astype(np.float64), gt + eq_before


def sharded_mrr_score(model, test, train=None, user_block=2048):
    """Collective ``evaluation.mrr_score`` of a :class:`ShardedImplicitFactorizationModel`: every rank
    calls it with the same arguments and gets the whole result.  Each rank ranks the test targets
    among its own item range (:meth:`ShardedImplicitFactorizationModel._eval_blocks`); the summed
    counts are those of the whole score row, so the result equals the single-GPU scorer's on the
    same tables, ties included, wherever the per-range GEMM reproduces the full GEMM's scores."""
    from spotlight_b200.interactions import _to_host
    test, train = _to_host(test), None if train is None else _to_host(train)
    n_users = int((np.diff(test.tocsr().indptr) > 0).sum())
    out = np.empty(n_users, dtype=np.float64)
    for lo, te, counts in model._eval_blocks(test, train, user_block):
        ranks, _ = _finalize_ranks(counts)
        n_per = np.diff(te.indptr)
        sums = np.add.reduceat(1.0 / ranks, te.indptr[:-1])
        out[lo:lo + len(n_per)] = sums / n_per
    return out


def sharded_precision_recall_score(model, test, train=None, k=10, user_block=2048):
    """Collective ``evaluation.precision_recall_score`` of a :class:`ShardedImplicitFactorizationModel`
    (see :func:`sharded_mrr_score`): precision = hits / min(k, num_items) with the global number of
    items, recall = hits / the user's number of test items; ties across the k boundary ordered by
    ascending item id."""
    from spotlight_b200.evaluation import _hits_at
    from spotlight_b200.interactions import _to_host
    test, train = _to_host(test), None if train is None else _to_host(train)
    ks = np.array([k]) if np.isscalar(k) else np.asarray(k)
    n_users = int((np.diff(test.tocsr().indptr) > 0).sum())
    hits = np.empty((n_users, len(ks)), dtype=np.int64)
    n_test = np.empty(n_users, dtype=np.int64)
    for lo, te, counts in model._eval_blocks(test, train, user_block):
        _, pos = _finalize_ranks(counts)
        n = len(te.indptr) - 1
        hits[lo:lo + n] = _hits_at(pos, te.indptr, ks)
        n_test[lo:lo + n] = np.diff(te.indptr)
    precision = hits / np.minimum(ks, model._num_items).reshape(1, -1).astype(np.float64)
    recall = hits / n_test.reshape(-1, 1).astype(np.float64)
    return precision.squeeze(), recall.squeeze()


def sharded_sequence_mrr_score(model, test, exclude_preceding=False, sequence_block=256):
    """Collective ``evaluation.sequence_mrr_score`` of a :class:`ShardedImplicitSequenceModel`: every
    rank calls it with the same arguments and gets the whole result.  Each rank ranks the last item
    of every test sequence among its own item range (:meth:`ShardedImplicitSequenceModel._eval_blocks`);
    the summed counts are those of the whole score row, so the result equals the single-GPU scorer's
    on ``gathered_net()``, ties included, wherever the per-range scores reproduce the full row's."""
    from spotlight_b200.evaluation import _check_items
    from spotlight_b200.interactions import _to_host
    test = _to_host(test)
    _check_items(test.sequences.reshape(-1), model._num_items)
    sequences = test.sequences[:, :-1]
    out = np.empty(len(sequences), dtype=np.float64)
    for lo, counts in model._eval_blocks(sequences, test.sequences[:, -1:].astype(np.int64), exclude_preceding,
                                         sequence_block):
        ranks, _ = _finalize_ranks(counts)
        out[lo:lo + len(ranks)] = 1.0 / ranks
    return out


def sharded_sequence_precision_recall_score(model, test, k=10, exclude_preceding=False, sequence_block=256):
    """Collective ``evaluation.sequence_precision_recall_score`` of a
    :class:`ShardedImplicitSequenceModel` (see :func:`sharded_sequence_mrr_score`): hits count the
    distinct targets among the last k items ranked in the top k; precision = hits / min(k,
    num_items), recall = hits / k; ties across the k boundary ordered by ascending item id."""
    from spotlight_b200.evaluation import _check_items, _hits_at
    from spotlight_b200.interactions import _to_host
    test = _to_host(test)
    S = test.sequences.shape[1]
    if not 0 < k < S:
        raise ValueError('k = %d must be in [1, sequence length %d)' % (k, S))
    _check_items(test.sequences.reshape(-1), model._num_items)
    sequences = test.sequences[:, :-k]
    targets = np.sort(test.sequences[:, -k:].astype(np.int64), axis=1)
    unique = np.ones(targets.shape, dtype=bool)
    unique[:, 1:] = targets[:, 1:] != targets[:, :-1]
    hits = np.empty(len(sequences), dtype=np.int64)
    for lo, counts in model._eval_blocks(sequences, targets, exclude_preceding, sequence_block):
        _, pos = _finalize_ranks(counts)
        n = len(pos) // k
        hits[lo:lo + n] = _hits_at(pos, np.arange(n + 1) * k, [k], unique[lo:lo + n].reshape(-1))[:, 0]
    return hits / float(min(k, model._num_items)), hits / float(k)
