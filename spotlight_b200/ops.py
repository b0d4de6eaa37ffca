"""PyTorch custom ops over the C-ABI library.

Each op replaces a span of the reference's hot path (citations in
include/spotlight_b200.h) and is registered with ``torch.library`` so that
``loss.backward()`` and any ``torch.optim`` optimizer keep working
(the reference's autograd/optimizer protocol,
spotlight/factorization/implicit.py:237-243).

PyTorch is plumbing here: it owns device memory and streams; all arithmetic
happens in the hand-written sm_90a kernels.  CPU tensors are rejected -- there
is no CPU path.
"""

import ctypes
from typing import List, Optional, Tuple

import torch
from torch import Tensor

from spotlight_b200 import _lib
from spotlight_b200._lib import LOSS_KIND, MfBloomArgs, MfStepArgs, SeqStepArgs

# ---------------------------------------------------------------------------
# plumbing
# ---------------------------------------------------------------------------


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t: Optional[Tensor]):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def require_cuda(*tensors):
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise RuntimeError(
                'spotlight_b200 ops need CUDA tensors (sm_90a); there is no CPU path. '
                'Construct the model with use_cuda=True.')
        if t is not None and t.device.index != torch.cuda.current_device():
            # the library launches on the current device and never calls cudaSetDevice
            raise RuntimeError(
                'spotlight_b200 ops launch on the current CUDA device (cuda:%d) but were given a tensor '
                'on %s; call torch.cuda.set_device(...) first (one process per GPU).'
                % (torch.cuda.current_device(), t.device))


def _f32c(t: Tensor) -> Tensor:
    if t.dtype != torch.float32:
        raise TypeError('spotlight_b200: parameters must be float32, got %s' % t.dtype)
    return t if t.is_contiguous() else t.contiguous()


def _i64c(t: Tensor) -> Tensor:
    if t.dtype != torch.int64:
        t = t.long()
    return t if t.is_contiguous() else t.contiguous()


_WORKSPACES = {}


def workspace(kind: str, nbytes: int, device) -> Tensor:
    """Persistent zero-initialised workspace, keyed by (kind, device, stream).

    The library keeps its scratch counters zero-at-rest, so a workspace is
    zeroed once and then reused; it grows geometrically.
    """
    dev = torch.device(device)
    key = (kind, dev.index if dev.index is not None else torch.cuda.current_device(),
           torch.cuda.current_stream(dev).cuda_stream)
    ws = _WORKSPACES.get(key)
    if ws is None or ws.numel() < nbytes:
        size = int(nbytes * 1.25) + 4096
        ws = torch.zeros(size, dtype=torch.uint8, device=dev)
        _WORKSPACES[key] = ws
    return ws


def workspace_error_word(ws: Tensor) -> Tensor:
    """The device-side id-range error word of an MF or row-bucketing workspace (int32 word 4 of
    the flags the library carves first), as a one-element view: nonzero once a kernel met an id
    outside its table."""
    return ws[:32].view(torch.int32)[4:5]


def workspace_error_flag(ws: Tensor) -> int:
    """Device-side id-range error flag of an MF workspace (workspace_error_word); reading clears
    it, so one bad batch does not poison later calls that share the cached workspace."""
    word = workspace_error_word(ws)
    flag = int(word.item())
    if flag:
        word.zero_()
    return flag


def _seeds_array(seeds):
    arr = (ctypes.c_uint32 * max(1, len(seeds)))(*[int(s) & 0xFFFFFFFF for s in seeds])
    return arr


# ---------------------------------------------------------------------------
# E1/E2/E3 embedding lookup (+ Bloom)        spotlight/layers.py:23-56,206-244
# ---------------------------------------------------------------------------

@torch.library.custom_op('spotlight_b200::embedding', mutates_args=())
def embedding(W: Tensor, ids: Tensor, seeds: List[int], padding_idx: int) -> Tensor:
    """out[n, D] = W[ids] (seeds == []) or sum_k W[murmur3(ids, seeds[k]) mod rows]."""
    require_cuda(W, ids)
    lib = _lib.load()
    W = _f32c(W)
    flat = _i64c(ids).reshape(-1)
    out = torch.empty((flat.numel(), W.shape[1]), dtype=torch.float32, device=W.device)
    rc = lib.slb_embedding_forward(_ptr(W), W.shape[0], W.shape[1], _ptr(flat), flat.numel(),
                                   len(seeds), _seeds_array(seeds), padding_idx, _ptr(out), _stream())
    _lib.check(rc, 'embedding_forward')
    return out


@embedding.register_fake
def _(W, ids, seeds, padding_idx):
    return W.new_empty((ids.numel(), W.shape[1]))


@torch.library.custom_op('spotlight_b200::embedding_backward', mutates_args=())
def embedding_backward(dout: Tensor, ids: Tensor, seeds: List[int], rows: int,
                       padding_idx: int) -> Tensor:
    """Deterministic segmented scatter-add of dout rows into a dense (rows, D) grad."""
    require_cuda(dout, ids)
    lib = _lib.load()
    dout = _f32c(dout)
    flat = _i64c(ids).reshape(-1)
    D = dout.shape[1]
    dW = torch.zeros((rows, D), dtype=torch.float32, device=dout.device)
    fan = max(1, len(seeds))
    need = lib.slb_embedding_backward_workspace_bytes(flat.numel() * fan, rows)
    ws = workspace('emb%d' % rows, need, dout.device)
    rc = lib.slb_embedding_backward(_ptr(dout), _ptr(flat), flat.numel(), len(seeds),
                                    _seeds_array(seeds), rows, D, padding_idx, _ptr(dW),
                                    _ptr(ws), ws.numel(), _stream())
    _lib.check(rc, 'embedding_backward')
    return dW


@embedding_backward.register_fake
def _(dout, ids, seeds, rows, padding_idx):
    return dout.new_empty((rows, dout.shape[1]))


def _embedding_setup(ctx, inputs, output):
    W, ids, seeds, padding_idx = inputs
    ctx.save_for_backward(ids)
    ctx.seeds = list(seeds)
    ctx.rows = W.shape[0]
    ctx.padding_idx = padding_idx


def _embedding_bwd(ctx, grad_out):
    (ids,) = ctx.saved_tensors
    dW = embedding_backward(grad_out.contiguous(), ids, ctx.seeds, ctx.rows, ctx.padding_idx)
    return dW, None, None, None


embedding.register_autograd(_embedding_bwd, setup_context=_embedding_setup)


@torch.library.custom_op('spotlight_b200::bloom_rows', mutates_args=())
def bloom_rows(ids: Tensor, seeds: List[int], rows: int, padding_idx: int) -> Tensor:
    """Hashed row ids (n, H) int64 -- BloomEmbedding._get_hashed_indices (layers.py:178-204)."""
    require_cuda(ids)
    lib = _lib.load()
    flat = _i64c(ids).reshape(-1)
    out = torch.empty((flat.numel(), len(seeds)), dtype=torch.int64, device=ids.device)
    rc = lib.slb_bloom_rows(_ptr(flat), flat.numel(), len(seeds), _seeds_array(seeds), rows,
                            padding_idx, _ptr(out), _stream())
    _lib.check(rc, 'bloom_rows')
    return out


# ---------------------------------------------------------------------------
# N1 BilinearNet.forward       spotlight/factorization/representations.py:80-91
# ---------------------------------------------------------------------------

@torch.library.custom_op('spotlight_b200::mf_scores', mutates_args=())
def mf_scores(Wu: Tensor, Wi: Tensor, bu: Tensor, bi: Tensor, users: Tensor,
              items: Tensor) -> Tensor:
    """scores[n] = <Wu[u], Wi[i]> + bu[u] + bi[i]; users may be a single id (broadcast)."""
    require_cuda(Wu, Wi, bu, bi, users, items)
    lib = _lib.load()
    users = _i64c(users).reshape(-1)
    items = _i64c(items).reshape(-1)
    n = items.numel()
    bcast = 1 if users.numel() == 1 and n != 1 else 0
    if not bcast and users.numel() != n:
        raise ValueError('mf_scores: users and items must have the same length')
    out = torch.empty(n, dtype=torch.float32, device=Wu.device)
    rc = lib.slb_mf_scores(_ptr(_f32c(Wu)), _ptr(_f32c(Wi)), _ptr(_f32c(bu)), _ptr(_f32c(bi)),
                           Wu.shape[1], _ptr(users), _ptr(items), n, bcast, _ptr(out), _stream())
    _lib.check(rc, 'mf_scores')
    return out


@mf_scores.register_fake
def _(Wu, Wi, bu, bi, users, items):
    return Wu.new_empty((items.numel(),))


@torch.library.custom_op('spotlight_b200::mf_scores_backward', mutates_args=())
def mf_scores_backward(g: Tensor, Wu: Tensor, Wi: Tensor, users: Tensor,
                       items: Tensor) -> Tuple[Tensor, Tensor, Tensor, Tensor]:
    require_cuda(g, Wu, Wi, users, items)
    lib = _lib.load()
    users = _i64c(users).reshape(-1)
    items = _i64c(items).reshape(-1)
    n = items.numel()
    bcast = 1 if users.numel() == 1 and n != 1 else 0
    U, D = Wu.shape
    I = Wi.shape[0]
    dWu = torch.zeros_like(Wu)
    dWi = torch.zeros_like(Wi)
    dbu = torch.zeros((U, 1), dtype=torch.float32, device=Wu.device)
    dbi = torch.zeros((I, 1), dtype=torch.float32, device=Wu.device)
    need = lib.slb_mf_step_workspace_bytes((n + 1) // 2, 1, 0, U, I)
    ws = workspace('mf%d_%d' % (U, I), need, Wu.device)
    rc = lib.slb_mf_scores_backward(_ptr(_f32c(g)), _ptr(users), _ptr(items), n, bcast,
                                    _ptr(_f32c(Wu)), _ptr(_f32c(Wi)), U, I, D,
                                    _ptr(dWu), _ptr(dWi), _ptr(dbu), _ptr(dbi),
                                    _ptr(ws), ws.numel(), _stream())
    _lib.check(rc, 'mf_scores_backward')
    return dWu, dWi, dbu, dbi


@mf_scores_backward.register_fake
def _(g, Wu, Wi, users, items):
    return (torch.empty_like(Wu), torch.empty_like(Wi),
            Wu.new_empty((Wu.shape[0], 1)), Wi.new_empty((Wi.shape[0], 1)))


def _mf_scores_setup(ctx, inputs, output):
    Wu, Wi, bu, bi, users, items = inputs
    ctx.save_for_backward(Wu, Wi, users, items)
    ctx.bshape = (bu.shape, bi.shape)


def _mf_scores_bwd(ctx, g):
    Wu, Wi, users, items = ctx.saved_tensors
    dWu, dWi, dbu, dbi = mf_scores_backward(g.contiguous(), Wu, Wi, users, items)
    return dWu, dWi, dbu.reshape(ctx.bshape[0]), dbi.reshape(ctx.bshape[1]), None, None


mf_scores.register_autograd(_mf_scores_bwd, setup_context=_mf_scores_setup)


# ---------------------------------------------------------------------------
# fused training step       spotlight/factorization/implicit.py:229-242
# ---------------------------------------------------------------------------

def mf_step_args(Wu, Wi, bu, bi, users, items, negs, loss, n_neg, batch=None, ratings=None):
    """A filled ``slb_mf_step_args`` (parameters + minibatch); caller adds outputs.
    Rating losses pass ``negs=None`` and the float32 ``ratings``."""
    a = MfStepArgs()
    a.batch = int(batch if batch is not None else users.numel())
    a.users, a.items = users.data_ptr(), items.data_ptr()
    a.negs = negs.data_ptr() if negs is not None else None
    a.ratings = ratings.data_ptr() if ratings is not None else None
    a.loss = LOSS_KIND[loss] if isinstance(loss, str) else int(loss)
    a.n_neg = int(n_neg)
    a.num_users, a.num_items, a.dim = Wu.shape[0], Wi.shape[0], Wu.shape[1]
    a.Wu, a.Wi, a.bu, a.bi = Wu.data_ptr(), Wi.data_ptr(), bu.data_ptr(), bi.data_ptr()
    return a


@torch.library.custom_op('spotlight_b200::mf_train_step', mutates_args=())
def mf_train_step(Wu: Tensor, Wi: Tensor, bu: Tensor, bi: Tensor, users: Tensor, items: Tensor,
                  negs: Tensor, loss: int, n_neg: int, want_scores: bool
                  ) -> Tuple[Tensor, Tensor, Tensor, Tensor, Tensor, Tensor, Tensor]:
    """Fused forward + backward of one minibatch with dense gradients.

    Returns (loss, pos, neg, dWu, dWi, dbu, dbi); pos/neg are empty unless
    ``want_scores``.  The gradients are those of ``loss`` itself (grad_output 1).
    """
    require_cuda(Wu, Wi, bu, bi, users, items, negs)
    lib = _lib.load()
    Wu, Wi, bu, bi = _f32c(Wu), _f32c(Wi), _f32c(bu), _f32c(bi)
    users, items, negs = _i64c(users).reshape(-1), _i64c(items).reshape(-1), _i64c(negs).reshape(-1)
    B = users.numel()
    if items.numel() != B or negs.numel() != B * n_neg:
        raise ValueError('mf_train_step: inconsistent batch sizes')
    dev = Wu.device
    a = mf_step_args(Wu, Wi, bu, bi, users, items, negs, loss, n_neg)
    loss_out = torch.empty(1, dtype=torch.float32, device=dev)
    pos = torch.empty(B if want_scores else 0, dtype=torch.float32, device=dev)
    neg = torch.empty(B * n_neg if want_scores else 0, dtype=torch.float32, device=dev)
    dWu, dWi = torch.zeros_like(Wu), torch.zeros_like(Wi)
    dbu, dbi = torch.zeros_like(bu), torch.zeros_like(bi)
    a.loss_out = loss_out.data_ptr()
    if want_scores:
        a.pos_out, a.neg_out = pos.data_ptr(), neg.data_ptr()
    a.grad_mode = _lib.GRAD_DENSE
    a.dWu, a.dWi, a.dbu, a.dbi = dWu.data_ptr(), dWi.data_ptr(), dbu.data_ptr(), dbi.data_ptr()
    need = lib.slb_mf_step_workspace_bytes(B, n_neg, a.loss, a.num_users, a.num_items)
    ws = workspace('mf%d_%d' % (a.num_users, a.num_items), need, dev)
    a.workspace, a.workspace_bytes = ws.data_ptr(), ws.numel()
    _lib.check(lib.slb_mf_train_step(ctypes.byref(a), _stream()), 'mf_train_step')
    return loss_out.reshape(()), pos, neg, dWu, dWi, dbu, dbi


@mf_train_step.register_fake
def _(Wu, Wi, bu, bi, users, items, negs, loss, n_neg, want_scores):
    B = users.numel()
    return (Wu.new_empty(()), Wu.new_empty((B if want_scores else 0,)),
            Wu.new_empty((B * n_neg if want_scores else 0,)),
            torch.empty_like(Wu), torch.empty_like(Wi), torch.empty_like(bu), torch.empty_like(bi))


def _adam_scalars(a, beta1, beta2, sched, step):
    """The lazy-exact Adam scalars of an MF, hashed-table or sequence step's arguments (the structs
    share the field names): ``1 - beta`` is taken in double, as torch's Python does, and ``sched``
    is ``FusedAdam.schedule``'s table reaching step ``step``."""
    b1, b2 = float(beta1), float(beta2)
    a.beta1, a.beta2, a.one_minus_beta1, a.one_minus_beta2 = b1, b2, 1.0 - b1, 1.0 - b2
    a.adam_sched, a.adam_step = sched.data_ptr(), int(step)


def v2_eligible(a):
    """Whether the step ``a`` (optimizer filled in) runs the planned two-kernel step (csrc/mf_v2.cuh)
    once it is given the fused workspace: the host's side of ``v2_eligible`` in csrc/mf.cu.  Adaptive
    hinge and lazy-exact Adam run the first-generation kernels, and so does a width for which
    slb_mf_fused_workspace_bytes is 0."""
    return a.loss != LOSS_KIND['adaptive_hinge'] and a.opt in (_lib.OPT_SGD, _lib.OPT_ADAGRAD)


def _mf_workspaces(a, dev, planned=True):
    """(step workspace, fused workspace) of the step ``a``: the fused one only for the planned step
    (``planned``, :func:`v2_eligible` and a width the library has one for), else None."""
    lib = _lib.load()
    need2 = (lib.slb_mf_fused_workspace_bytes(a.batch, a.num_users, a.num_items, a.dim)
             if planned and v2_eligible(a) else 0)
    fws = workspace('mfv2_%d_%d_%d' % (a.num_users, a.num_items, a.dim), need2, dev) if need2 else None
    ws = workspace('mf%d_%d' % (a.num_users, a.num_items),
                   lib.slb_mf_step_workspace_bytes(a.batch, a.n_neg, a.loss, a.num_users, a.num_items), dev)
    return ws, fws


def mf_fused_step_args(Wu, Wi, bu, bi, users, items, negs, loss, n_neg, opt_kind, hp, states, batch=None,
                       ratings=None, adam=None, planned=True):
    """A filled ``slb_mf_step_args`` for steps with the row-wise optimizer fused in: both tables
    take their update in place through compact gradients.  ``hp`` = dict(lr, weight_decay, eps)
    (``fused_hparams()``); ``states`` = Adagrad's (sWu, sWi, sbu, sbi), or under lazy-exact Adam
    four (exp_avg, exp_avg_sq, last) of (Wu, Wi, bu, bi) with ``adam`` = dict(beta1, beta2, sched,
    step (the first step, 1-based)).

    The planned step gets its fused workspace when ``planned`` and :func:`v2_eligible` allow and
    the library has a workspace for the width; otherwise the first-generation step gets its seven
    compact buffers.  Returns (args, ws, keep): the caller sets ``loss_out`` (and ``plan_stream``)
    and launches, reads the id-range flag of the workspace ``ws`` (workspace_error_flag), and holds
    ``keep`` until the launch is enqueued."""
    lib = _lib.load()
    dev = Wu.device
    a = mf_step_args(Wu, Wi, bu, bi, users, items, negs, loss, n_neg, batch=batch, ratings=ratings)
    a.grad_mode = _lib.GRAD_COMPACT
    a.opt, a.lr, a.weight_decay, a.eps = int(opt_kind), float(hp['lr']), float(hp['weight_decay']), float(hp['eps'])
    keep = []
    if opt_kind == _lib.OPT_ADAGRAD:
        a.state_Wu, a.state_Wi, a.state_bu, a.state_bi = [t.data_ptr() for t in states]
    elif opt_kind == _lib.OPT_ADAM:
        a.state_Wu, a.state_Wi, a.state_bu, a.state_bi = [s[0].data_ptr() for s in states]
        a.state2_Wu, a.state2_Wi, a.state2_bu, a.state2_bi = [s[1].data_ptr() for s in states]
        a.last_u, a.last_i = states[0][2].data_ptr(), states[1][2].data_ptr()
        _adam_scalars(a, adam['beta1'], adam['beta2'], adam['sched'], adam['step'])
        keep.append(adam['sched'])
    ws, fws = _mf_workspaces(a, dev, planned)
    a.workspace, a.workspace_bytes = ws.data_ptr(), ws.numel()
    if fws is not None:
        a.fused_workspace, a.fused_workspace_bytes = fws.data_ptr(), fws.numel()
    else:
        rows = lib.slb_mf_compact_rows(a.batch, a.n_neg, a.loss, 0)
        bufs = [torch.empty(rows, dtype=torch.int64, device=dev), torch.empty(rows, dtype=torch.int64, device=dev),
                torch.empty((rows, a.dim), device=dev), torch.empty((rows, a.dim), device=dev),
                torch.empty(rows, device=dev), torch.empty(rows, device=dev),
                torch.zeros(2, dtype=torch.int32, device=dev)]
        a.urows, a.irows, a.gWu, a.gWi, a.gbu, a.gbi, a.compact_counts = [t.data_ptr() for t in bufs]
        keep += bufs
    return a, ws, keep


def mf_train_step_inplace(Wu, Wi, bu, bi, users, items, negs, loss, opt_kind, lr, states=None,
                          weight_decay=0.0, eps=1e-10, planned=True, ratings=None):
    """One minibatch with the row-wise optimizer fused in: parameters (and Adagrad ``states`` =
    (sWu, sWi, sbu, sbi)) are updated in place, the minibatch loss is returned.

    ``planned`` selects the two-kernel planned step (csrc/mf_v2.cuh) when the library supports
    the shape; otherwise the first-generation step with compact gradients runs.  This is the
    body of one iteration of ``slb_mf_fit_epoch`` (spotlight/factorization/implicit.py:229-243).
    Rating losses pass ``negs=None`` and ``ratings`` (spotlight/factorization/explicit.py:223-234).
    """
    require_cuda(Wu, Wi, bu, bi, users, items, negs, ratings)
    users, items = _i64c(users).reshape(-1), _i64c(items).reshape(-1)
    negs = _i64c(negs).reshape(-1) if negs is not None else None
    ratings = _f32c(ratings).reshape(-1) if ratings is not None else None
    with torch.no_grad():
        a, _, keep = mf_fused_step_args(Wu, Wi, bu, bi, users, items, negs, loss, 1, opt_kind,
                                        dict(lr=lr, weight_decay=weight_decay, eps=eps), states,
                                        ratings=ratings, planned=planned)
        loss_out = torch.empty(1, dtype=torch.float32, device=Wu.device)
        a.loss_out = loss_out.data_ptr()
        _lib.check(_lib.load().slb_mf_train_step(ctypes.byref(a), _stream()), 'mf_train_step')
    return loss_out.reshape(())


def _bloom_args(Wu, Wi, bu, bi, users, items, negs, ratings, loss, n_neg, user_seeds, item_seeds, user_pad,
                item_pad):
    """A filled ``slb_mf_bloom_args`` (tables, hashes, minibatch); the caller adds outputs and the
    optimizer, then :func:`_bloom_workspace`.  Pairwise losses pass ``negs``, rating losses
    ``ratings`` (the other None)."""
    x = MfBloomArgs()
    a = x.base
    a.batch = users.numel()
    a.users, a.items = users.data_ptr(), items.data_ptr()
    a.negs = negs.data_ptr() if negs is not None else None
    a.ratings = ratings.data_ptr() if ratings is not None else None
    a.loss = LOSS_KIND[loss] if isinstance(loss, str) else int(loss)
    a.n_neg = int(n_neg)
    a.num_users, a.num_items, a.dim = bu.shape[0], bi.shape[0], Wu.shape[1]
    a.Wu, a.Wi, a.bu, a.bi = Wu.data_ptr(), Wi.data_ptr(), bu.data_ptr(), bi.data_ptr()
    x.user_rows, x.item_rows = Wu.shape[0], Wi.shape[0]
    x.user_hashes, x.item_hashes = len(user_seeds), len(item_seeds)
    for k, sd in enumerate(user_seeds):
        x.user_seeds[k] = int(sd) & 0xFFFFFFFF
    for k, sd in enumerate(item_seeds):
        x.item_seeds[k] = int(sd) & 0xFFFFFFFF
    x.user_padding_idx, x.item_padding_idx = int(user_pad), int(item_pad)
    return x


def _bloom_workspace(kind, x, dev):
    """Attach the workspace of ``x``: one per (kind, shapes, hash counts, loss family, batch),
    because its zero-at-rest regions are layout dependent and a rating loss lays out one scored
    side per interaction where a pairwise loss lays out two."""
    a = x.base
    family = 'rating' if a.loss >= LOSS_KIND['regression'] else 'pairwise'
    ws = workspace('%s_%s_%d_%d_%d_%d_%d_%d_%d' % (kind, family, x.user_rows, x.item_rows, a.num_users, a.num_items,
                                                   x.user_hashes, x.item_hashes, a.batch),
                   _lib.load().slb_mf_bloom_workspace_bytes(ctypes.byref(x)), dev)
    a.workspace, a.workspace_bytes = ws.data_ptr(), ws.numel()
    return ws


def _bloom_dense_step(Wu, Wi, bu, bi, users, items, negs, ratings, loss, n_neg, user_seeds, item_seeds,
                      user_pad, item_pad, want_scores):
    """The hashed-table step with dense gradients: (loss, pos, neg, dWu, dWi, dbu, dbi)."""
    Wu, Wi, bu, bi = _f32c(Wu), _f32c(Wi), _f32c(bu), _f32c(bi)
    B = users.numel()
    dev = Wu.device
    x = _bloom_args(Wu, Wi, bu, bi, users, items, negs, ratings, loss, n_neg, user_seeds, item_seeds, user_pad,
                    item_pad)
    a = x.base
    loss_out = torch.empty(1, dtype=torch.float32, device=dev)
    pos = torch.empty(B if want_scores else 0, dtype=torch.float32, device=dev)
    neg = torch.empty(B * n_neg if want_scores and negs is not None else 0, dtype=torch.float32, device=dev)
    dWu, dWi = torch.zeros_like(Wu), torch.zeros_like(Wi)
    dbu, dbi = torch.zeros_like(bu), torch.zeros_like(bi)
    a.loss_out = loss_out.data_ptr()
    if want_scores:
        a.pos_out = pos.data_ptr()
        a.neg_out = neg.data_ptr() if negs is not None else None
    a.grad_mode = _lib.GRAD_DENSE
    a.dWu, a.dWi, a.dbu, a.dbi = dWu.data_ptr(), dWi.data_ptr(), dbu.data_ptr(), dbi.data_ptr()
    _bloom_workspace('mfb', x, dev)
    _lib.check(_lib.load().slb_mf_bloom_train_step(ctypes.byref(x), _stream()), 'mf_bloom_train_step')
    return loss_out.reshape(()), pos, neg, dWu, dWi, dbu, dbi


@torch.library.custom_op('spotlight_b200::mf_bloom_train_step', mutates_args=())
def mf_bloom_train_step(Wu: Tensor, Wi: Tensor, bu: Tensor, bi: Tensor, users: Tensor, items: Tensor,
                        negs: Tensor, loss: int, n_neg: int, user_seeds: List[int],
                        item_seeds: List[int], user_pad: int, item_pad: int, want_scores: bool
                        ) -> Tuple[Tensor, Tensor, Tensor, Tensor, Tensor, Tensor, Tensor]:
    """Fused step for BilinearNet with BloomEmbedding user / item layers (empty seed list
    = plain table).  Wu / Wi are the (hashed) embedding tables, bu / bi the id-indexed
    biases.  Returns (loss, pos, neg, dWu, dWi, dbu, dbi), dense."""
    require_cuda(Wu, Wi, bu, bi, users, items, negs)
    users, items, negs = _i64c(users).reshape(-1), _i64c(items).reshape(-1), _i64c(negs).reshape(-1)
    B = users.numel()
    if items.numel() != B or negs.numel() != B * n_neg:
        raise ValueError('mf_bloom_train_step: inconsistent batch sizes')
    return _bloom_dense_step(Wu, Wi, bu, bi, users, items, negs, None, loss, n_neg, user_seeds, item_seeds,
                             user_pad, item_pad, want_scores)


@mf_bloom_train_step.register_fake
def _(Wu, Wi, bu, bi, users, items, negs, loss, n_neg, user_seeds, item_seeds, user_pad, item_pad,
      want_scores):
    B = users.numel()
    return (Wu.new_empty(()), Wu.new_empty((B if want_scores else 0,)),
            Wu.new_empty((B * n_neg if want_scores else 0,)),
            torch.empty_like(Wu), torch.empty_like(Wi), torch.empty_like(bu), torch.empty_like(bi))


@torch.library.custom_op('spotlight_b200::mf_bloom_rating_step', mutates_args=())
def mf_bloom_rating_step(Wu: Tensor, Wi: Tensor, bu: Tensor, bi: Tensor, users: Tensor, items: Tensor,
                         ratings: Tensor, loss: int, user_seeds: List[int], item_seeds: List[int], user_pad: int,
                         item_pad: int, want_scores: bool
                         ) -> Tuple[Tensor, Tensor, Tensor, Tensor, Tensor, Tensor]:
    """Fused explicit-feedback step (regression / poisson / logistic) for BilinearNet with
    BloomEmbedding user / item layers (empty seed list = plain table), dense gradients.
    Returns (loss, scores, dWu, dWi, dbu, dbi); ``scores`` (the raw BilinearNet output) is empty
    unless ``want_scores``."""
    require_cuda(Wu, Wi, bu, bi, users, items, ratings)
    users, items = _i64c(users).reshape(-1), _i64c(items).reshape(-1)
    ratings = _f32c(ratings).reshape(-1)
    B = users.numel()
    if items.numel() != B or ratings.numel() != B:
        raise ValueError('mf_bloom_rating_step: inconsistent batch sizes')
    out = _bloom_dense_step(Wu, Wi, bu, bi, users, items, None, ratings, loss, 1, user_seeds, item_seeds,
                            user_pad, item_pad, want_scores)
    return out[:2] + out[3:]


@mf_bloom_rating_step.register_fake
def _(Wu, Wi, bu, bi, users, items, ratings, loss, user_seeds, item_seeds, user_pad, item_pad, want_scores):
    B = users.numel()
    return (Wu.new_empty(()), Wu.new_empty((B if want_scores else 0,)),
            torch.empty_like(Wu), torch.empty_like(Wi), torch.empty_like(bu), torch.empty_like(bi))


def mf_bloom_train_step_inplace(Wu, Wi, bu, bi, users, items, negs, loss, n_neg, user_seeds, item_seeds,
                                user_pad, item_pad, opt_kind, lr, states=None, weight_decay=0.0, eps=1e-10,
                                ratings=None, adam=None):
    """The fused hashed-table step with the row-wise optimizer applied in place: hashed / plain
    embedding rows through the compact-gradient kernels, the id-indexed bias tables through the
    hash-bucket sparse update (no dense gradient anywhere -- the item-bias table of BASELINE
    config 4 has 50 M rows).  ``states`` = (sWu, sWi, sbu, sbi) for Adagrad.  Rating losses pass
    ``negs=None``, ``n_neg=1`` and ``ratings`` (spotlight/factorization/explicit.py:223-234).

    Lazy-exact Adam (``opt_kind = OPT_ADAM``, pairwise losses): ``states`` = four (exp_avg,
    exp_avg_sq, last) triples of (Wu, Wi, bu, bi) (``FusedAdam.fused_states(p, own_last=True)``; each
    ``last`` int32 with one entry per row), ``adam`` = dict(beta1, beta2, sched
    (``FusedAdam.schedule``), step (this step, 1-based)).  Every row and bias the minibatch reads is
    first brought current through step - 1; the entries with a gradient then take step.
    Returns the loss."""
    require_cuda(Wu, Wi, bu, bi, users, items, negs, ratings)
    users, items = _i64c(users).reshape(-1), _i64c(items).reshape(-1)
    negs = _i64c(negs).reshape(-1) if negs is not None else None
    ratings = _f32c(ratings).reshape(-1) if ratings is not None else None
    dev = Wu.device
    with torch.no_grad():
        x = _bloom_args(Wu, Wi, bu, bi, users, items, negs, ratings, loss, n_neg, user_seeds, item_seeds, user_pad,
                        item_pad)
        a = x.base
        loss_out = torch.empty(1, dtype=torch.float32, device=dev)
        a.loss_out = loss_out.data_ptr()
        a.grad_mode = _lib.GRAD_COMPACT
        a.opt, a.lr, a.weight_decay, a.eps = int(opt_kind), float(lr), float(weight_decay), float(eps)
        if opt_kind == _lib.OPT_ADAGRAD:
            a.state_Wu, a.state_Wi, a.state_bu, a.state_bi = [t.data_ptr() for t in states]
        elif opt_kind == _lib.OPT_ADAM:
            _bloom_adam_args(x, (Wu, Wi, bu, bi), states, adam)
        # the Adam layout adds compact user-row gradients: its own workspace
        _bloom_workspace('mfbfa' if opt_kind == _lib.OPT_ADAM else 'mfbf', x, dev)
        _lib.check(_lib.load().slb_mf_bloom_train_step(ctypes.byref(x), _stream()), 'mf_bloom_train_step')
    return loss_out.reshape(())


def _bloom_adam_args(x, params, states, adam):
    """The lazy-exact Adam fields of slb_mf_bloom_args (see mf_bloom_train_step_inplace)."""
    if states is None or len(states) != 4 or adam is None:
        raise ValueError('mf_bloom_train_step: Adam needs four (exp_avg, exp_avg_sq, last) states and adam=')
    require_cuda(adam['sched'], *[t for st in states for t in st])
    for p, (m, v, last) in zip(params, states):
        for t in (m, v):
            if t.shape != p.shape or t.dtype != torch.float32 or not t.is_contiguous():
                raise ValueError('mf_bloom_train_step: Adam moments must be contiguous float32 of the parameter shape')
        if last.dtype != torch.int32 or last.shape != (p.shape[0],) or not last.is_contiguous():
            raise ValueError('mf_bloom_train_step: Adam `last` must be contiguous int32 with one entry per row')
    step = int(adam['step'])
    if adam['sched'].numel() < 2 * (step + 1):
        raise ValueError('mf_bloom_train_step: the Adam schedule does not reach step %d' % step)
    a = x.base
    a.state_Wu, a.state_Wi, a.state_bu, a.state_bi = [st[0].data_ptr() for st in states]
    a.state2_Wu, a.state2_Wi, a.state2_bu, a.state2_bi = [st[1].data_ptr() for st in states]
    a.last_u, a.last_i = states[0][2].data_ptr(), states[1][2].data_ptr()
    x.last_bu, x.last_bi = states[2][2].data_ptr(), states[3][2].data_ptr()
    _adam_scalars(a, adam['beta1'], adam['beta2'], adam['sched'], step)


def mf_bloom_step_pairs(Wu, Wi, bu, bi, users, items, negs, loss, item_seeds, item_pad, norm_batch=0,
                        users_only=None, dWi=None):
    """Dense-mode hashed-table step for the multi-GPU path: plain (local) user table, hashed item
    table given in full; returns (loss share, dWu, dWi, (ids_u, g_u), (ids_i, g_i)) -- the
    id-space bias gradients as (id, g) pairs instead of dense tables.

    ``users_only``: the user rows and user biases take their optimizer step in place instead
    (slb_mf_bloom_args' users-only mode; pointwise / bpr / hinge), and ``dWu`` and the user pairs
    come back as None.  dict(opt=OPT_ADAGRAD, lr, eps, states=(sWu, sbu)), or dict(opt=OPT_ADAM,
    lr, eps, weight_decay, beta1, beta2, sched, step, states=((mWu, vWu, last_u), (mbu, vbu),
    (mbi, vbi, last_bi))): the user rows and biases share ``last_u``; ``last_bi`` is this replica's
    item-bias ``last``.  ``dWi``: a zeroed (item_rows, D) buffer to write the item gradient to."""
    require_cuda(Wu, Wi, bu, bi, users, items, negs)
    lib = _lib.load()
    users, items, negs = _i64c(users).reshape(-1), _i64c(items).reshape(-1), _i64c(negs).reshape(-1)
    B = users.numel()
    dev = Wu.device
    with torch.no_grad():
        x = MfBloomArgs()
        a = x.base
        a.batch = B
        a.users, a.items, a.negs = users.data_ptr(), items.data_ptr(), negs.data_ptr()
        a.loss, a.n_neg = (LOSS_KIND[loss] if isinstance(loss, str) else int(loss)), 1
        a.num_users, a.num_items, a.dim = bu.shape[0], bi.shape[0], Wu.shape[1]
        a.Wu, a.Wi, a.bu, a.bi = Wu.data_ptr(), Wi.data_ptr(), bu.data_ptr(), bi.data_ptr()
        loss_out = torch.empty(1, dtype=torch.float32, device=dev)
        if dWi is None:
            dWi = torch.zeros_like(Wi)
        elif dWi.shape != Wi.shape or dWi.dtype != torch.float32 or not dWi.is_contiguous():
            raise ValueError('mf_bloom_step_pairs: dWi must be contiguous float32 of the item table\'s shape')
        pi_i = torch.empty(2 * B, dtype=torch.int64, device=dev)
        pi_g = torch.empty(2 * B, dtype=torch.float32, device=dev)
        a.loss_out = loss_out.data_ptr()
        a.grad_mode = _lib.GRAD_DENSE
        a.dWi = dWi.data_ptr()
        a.norm_batch = int(norm_batch)
        x.pair_ids_i, x.pair_g_i = pi_i.data_ptr(), pi_g.data_ptr()
        if users_only is None:
            dWu = torch.zeros_like(Wu)
            pu_i = torch.empty(2 * B, dtype=torch.int64, device=dev)
            pu_g = torch.empty(2 * B, dtype=torch.float32, device=dev)
            a.dWu = dWu.data_ptr()
            x.pair_ids_u, x.pair_g_u = pu_i.data_ptr(), pu_g.data_ptr()
            upairs = (pu_i, pu_g)
        else:
            dWu, upairs = None, None
            _bloom_users_only_args(x, users_only)
        x.user_rows, x.item_rows = Wu.shape[0], Wi.shape[0]
        x.user_hashes, x.item_hashes = 0, len(item_seeds)
        for k, sd in enumerate(item_seeds):
            x.item_seeds[k] = int(sd) & 0xFFFFFFFF
        x.user_padding_idx, x.item_padding_idx = -1, item_pad
        need = lib.slb_mf_bloom_workspace_bytes(ctypes.byref(x))
        kind = 'mfbp' if users_only is None else 'mfbu%d_' % a.opt
        ws = workspace(kind + '%d_%d_%d_%d_%d_%d' % (Wu.shape[0], Wi.shape[0], bu.shape[0], bi.shape[0],
                                                     len(item_seeds), B), need, dev)
        a.workspace, a.workspace_bytes = ws.data_ptr(), ws.numel()
        _lib.check(lib.slb_mf_bloom_train_step(ctypes.byref(x), _stream()), 'mf_bloom_train_step')
    return loss_out.reshape(()), dWu, dWi, upairs, (pi_i, pi_g)


def _bloom_users_only_args(x, uo):
    """The users-only fields of slb_mf_bloom_args (see mf_bloom_step_pairs)."""
    a = x.base
    a.opt, a.opt_users_only = int(uo['opt']), 1
    a.lr, a.eps, a.weight_decay = float(uo['lr']), float(uo['eps']), float(uo.get('weight_decay', 0.0))
    if uo['opt'] == _lib.OPT_ADAGRAD:
        sWu, sbu = uo['states']
        require_cuda(sWu, sbu)
        a.state_Wu, a.state_bu = sWu.data_ptr(), sbu.data_ptr()
        return
    (mWu, vWu, last_u), (mbu, vbu), (mbi, vbi, last_bi) = uo['states']
    require_cuda(mWu, vWu, last_u, mbu, vbu, mbi, vbi, last_bi, uo['sched'])
    step = int(uo['step'])
    if uo['sched'].numel() < 2 * (step + 1):
        raise ValueError('mf_bloom_step_pairs: the Adam schedule does not reach step %d' % step)
    a.state_Wu, a.state2_Wu, a.last_u = mWu.data_ptr(), vWu.data_ptr(), last_u.data_ptr()
    a.state_bu, a.state2_bu = mbu.data_ptr(), vbu.data_ptr()
    a.state_bi, a.state2_bi, x.last_bi = mbi.data_ptr(), vbi.data_ptr(), last_bi.data_ptr()
    _adam_scalars(a, uo['beta1'], uo['beta2'], uo['sched'], step)


def bias_sparse_adam(ids, g, bias, exp_avg, exp_avg_sq, last, sched, step, beta1, beta2, eps, weight_decay):
    """Lazy-exact Adam step ``step`` of an id-indexed bias table from (id, g) pairs
    (slb_bias_sparse_adam): each id with a pair (id >= 0) catches up from its ``last``, sums its
    pairs in pair order and takes the step."""
    require_cuda(ids, g, bias, exp_avg, exp_avg_sq, last, sched)
    lib = _lib.load()
    n = ids.numel()
    if n == 0:
        return
    ws = workspace('bsp%d' % n, lib.slb_bias_sparse_workspace_bytes(n), bias.device)
    ids, g = _i64c(ids), _f32c(g)           # held until the launch: a temporary's block could be reused
    with torch.no_grad():
        _lib.check(lib.slb_bias_sparse_adam(_ptr(ids), _ptr(g), n, _ptr(bias), _ptr(exp_avg),
                                            _ptr(exp_avg_sq), _ptr(last), _ptr(sched), int(step), float(beta1),
                                            float(beta2), 1.0 - float(beta1), 1.0 - float(beta2), float(eps),
                                            float(weight_decay), _ptr(ws), ws.numel(), _stream()),
                   'bias_sparse_adam')


def bias_sparse_apply(ids, g, bias, state, opt_kind, lr, weight_decay=0.0, eps=1e-10):
    """In-place SGD / Adagrad update of an id-indexed bias table from (id, g) pairs (g == 0 pairs
    are padding)."""
    require_cuda(ids, g, bias)
    lib = _lib.load()
    n = ids.numel()
    if n == 0:
        return
    ws = workspace('bsp%d' % n, lib.slb_bias_sparse_workspace_bytes(n), bias.device)
    with torch.no_grad():
        _lib.check(lib.slb_bias_sparse_apply(_ptr(_i64c(ids)), _ptr(_f32c(g)), n, _ptr(bias), _ptr(state),
                                             int(opt_kind), float(lr), float(weight_decay), float(eps),
                                             _ptr(ws), ws.numel(), _stream()), 'bias_sparse_apply')


class _FusedBloomLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, Wu, Wi, bu, bi, users, items, negs, loss, n_neg, us, its, up, ip):
        out = mf_bloom_train_step(Wu.detach(), Wi.detach(), bu.detach(), bi.detach(), users, items,
                                  negs, loss, n_neg, us, its, up, ip, False)
        ctx.save_for_backward(*out[3:])
        return out[0]

    @staticmethod
    def backward(ctx, g):
        dWu, dWi, dbu, dbi = ctx.saved_tensors
        return (dWu * g, dWi * g, dbu * g, dbi * g) + (None,) * 9


def fused_bloom_loss(Wu, Wi, bu, bi, users, items, negs, loss: str, n_neg, spec):
    """As :func:`fused_mf_loss` for hashed tables; ``spec`` from BilinearNet.fused_spec()."""
    return _FusedBloomLoss.apply(Wu, Wi, bu, bi, users, items, negs, LOSS_KIND[loss], n_neg,
                                 spec['user_seeds'], spec['item_seeds'], spec['user_pad'],
                                 spec['item_pad'])


class _FusedMFLoss(torch.autograd.Function):
    """loss = fused_step(...); backward hands out the gradients computed in forward."""

    @staticmethod
    def forward(ctx, Wu, Wi, bu, bi, users, items, negs, loss, n_neg):
        out = mf_train_step(Wu.detach(), Wi.detach(), bu.detach(), bi.detach(), users, items,
                            negs, loss, n_neg, False)
        ctx.save_for_backward(*out[3:])
        return out[0]

    @staticmethod
    def backward(ctx, g):
        dWu, dWi, dbu, dbi = ctx.saved_tensors
        return dWu * g, dWi * g, dbu * g, dbi * g, None, None, None, None, None


def fused_mf_loss(Wu, Wi, bu, bi, users, items, negs, loss: str, n_neg: int = 1):
    """Scalar minibatch loss whose ``backward()`` fills dense ``.grad`` on the
    four BilinearNet parameters (one fused kernel per direction)."""
    return _FusedMFLoss.apply(Wu, Wi, bu, bi, users, items, negs, LOSS_KIND[loss], n_neg)


# ---------------------------------------------------------------------------
# explicit-feedback step     spotlight/factorization/explicit.py:223-234
# ---------------------------------------------------------------------------

@torch.library.custom_op('spotlight_b200::mf_rating_train_step', mutates_args=())
def mf_rating_train_step(Wu: Tensor, Wi: Tensor, bu: Tensor, bi: Tensor, users: Tensor, items: Tensor,
                         ratings: Tensor, loss: int, want_scores: bool
                         ) -> Tuple[Tensor, Tensor, Tensor, Tensor, Tensor, Tensor]:
    """Fused forward + backward of one rating minibatch with dense gradients.

    Returns (loss, scores, dWu, dWi, dbu, dbi); ``scores`` (the raw BilinearNet output, before
    poisson's exp / logistic's sigmoid) is empty unless ``want_scores``.
    """
    require_cuda(Wu, Wi, bu, bi, users, items, ratings)
    lib = _lib.load()
    Wu, Wi, bu, bi = _f32c(Wu), _f32c(Wi), _f32c(bu), _f32c(bi)
    users, items = _i64c(users).reshape(-1), _i64c(items).reshape(-1)
    ratings = _f32c(ratings).reshape(-1)
    B = users.numel()
    if items.numel() != B or ratings.numel() != B:
        raise ValueError('mf_rating_train_step: inconsistent batch sizes')
    dev = Wu.device
    a = mf_step_args(Wu, Wi, bu, bi, users, items, None, loss, 1, ratings=ratings)
    loss_out = torch.empty(1, dtype=torch.float32, device=dev)
    pos = torch.empty(B if want_scores else 0, dtype=torch.float32, device=dev)
    dWu, dWi = torch.zeros_like(Wu), torch.zeros_like(Wi)
    dbu, dbi = torch.zeros_like(bu), torch.zeros_like(bi)
    a.loss_out = loss_out.data_ptr()
    if want_scores:
        a.pos_out = pos.data_ptr()
    a.grad_mode = _lib.GRAD_DENSE
    a.dWu, a.dWi, a.dbu, a.dbi = dWu.data_ptr(), dWi.data_ptr(), dbu.data_ptr(), dbi.data_ptr()
    need = lib.slb_mf_step_workspace_bytes(B, 1, a.loss, a.num_users, a.num_items)
    ws = workspace('mf%d_%d' % (a.num_users, a.num_items), need, dev)
    a.workspace, a.workspace_bytes = ws.data_ptr(), ws.numel()
    _lib.check(lib.slb_mf_train_step(ctypes.byref(a), _stream()), 'mf_rating_train_step')
    return loss_out.reshape(()), pos, dWu, dWi, dbu, dbi


@mf_rating_train_step.register_fake
def _(Wu, Wi, bu, bi, users, items, ratings, loss, want_scores):
    B = users.numel()
    return (Wu.new_empty(()), Wu.new_empty((B if want_scores else 0,)),
            torch.empty_like(Wu), torch.empty_like(Wi), torch.empty_like(bu), torch.empty_like(bi))


class _FusedRatingLoss(torch.autograd.Function):
    """loss = fused rating step(...); backward hands out the gradients computed in forward."""

    @staticmethod
    def forward(ctx, Wu, Wi, bu, bi, users, items, ratings, loss):
        out = mf_rating_train_step(Wu.detach(), Wi.detach(), bu.detach(), bi.detach(), users, items,
                                   ratings, loss, False)
        ctx.save_for_backward(*out[2:])
        return out[0]

    @staticmethod
    def backward(ctx, g):
        dWu, dWi, dbu, dbi = ctx.saved_tensors
        return dWu * g, dWi * g, dbu * g, dbi * g, None, None, None, None


def fused_rating_loss(Wu, Wi, bu, bi, users, items, ratings, loss: str):
    """Scalar minibatch rating loss whose ``backward()`` fills dense ``.grad`` on the four
    BilinearNet parameters: the body of the reference's explicit fit loop
    (explicit.py:223-233) in one fused kernel per direction."""
    return _FusedRatingLoss.apply(Wu, Wi, bu, bi, users, items, ratings, LOSS_KIND[loss])


# ---------------------------------------------------------------------------
# L1..L4 standalone losses                      spotlight/losses.py:18-166
# ---------------------------------------------------------------------------

@torch.library.custom_op('spotlight_b200::pairwise_loss', mutates_args=())
def pairwise_loss(pos: Tensor, neg: Tensor, mask: Optional[Tensor], loss: int
                  ) -> Tuple[Tensor, Tensor, Tensor]:
    """(loss, dloss/dpos, dloss/dneg).  neg is (n_neg, *pos.shape) for adaptive hinge."""
    require_cuda(pos, neg, mask)
    lib = _lib.load()
    p = _f32c(pos).reshape(-1)
    n = p.numel()
    ng = _f32c(neg).reshape(-1)
    n_neg = ng.numel() // max(n, 1)
    if n == 0 or ng.numel() != n * n_neg or (loss != 3 and n_neg != 1):
        raise ValueError('pairwise_loss: bad shapes pos %s neg %s' % (tuple(pos.shape), tuple(neg.shape)))
    m = None
    if mask is not None:
        m = mask.reshape(-1).to(torch.uint8).contiguous()
        if m.numel() != n:
            raise ValueError('pairwise_loss: mask shape mismatch')
    out = torch.empty(1, dtype=torch.float32, device=pos.device)
    gp = torch.empty_like(p)
    gn = torch.empty_like(ng)
    ws = workspace('loss', lib.slb_loss_workspace_bytes(n), pos.device)
    rc = lib.slb_pairwise_loss(loss, _ptr(p), _ptr(ng), _ptr(m), n, n_neg, _ptr(out), _ptr(gp),
                               _ptr(gn), _ptr(ws), ws.numel(), _stream())
    _lib.check(rc, 'pairwise_loss')
    return out.reshape(()), gp.reshape(pos.shape), gn.reshape(neg.shape)


@pairwise_loss.register_fake
def _(pos, neg, mask, loss):
    return pos.new_empty(()), torch.empty_like(pos), torch.empty_like(neg)


class _PairwiseLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pos, neg, mask, loss):
        l, gp, gn = pairwise_loss(pos.detach(), neg.detach(), mask, loss)
        ctx.save_for_backward(gp, gn)
        return l

    @staticmethod
    def backward(ctx, g):
        gp, gn = ctx.saved_tensors
        return gp * g, gn * g, None, None


def loss_op(kind: str, pos, neg, mask=None):
    return _PairwiseLoss.apply(pos, neg, mask, LOSS_KIND[kind])


# ---------------------------------------------------------------------------
# L5..L7 standalone rating losses                spotlight/losses.py:169-244
# ---------------------------------------------------------------------------

@torch.library.custom_op('spotlight_b200::rating_loss', mutates_args=())
def rating_loss(pred: Tensor, ratings: Tensor, loss: int) -> Tuple[Tensor, Tensor]:
    """(mean loss, d loss / d pred) of one rating loss; poisson takes the exponentiated
    prediction, as the reference's ``poisson_loss`` does."""
    require_cuda(pred, ratings)
    lib = _lib.load()
    p = _f32c(pred).reshape(-1)
    n = p.numel()
    r = ratings.reshape(-1).to(torch.float32).contiguous()
    if n == 0 or r.numel() != n:
        raise ValueError('rating_loss: bad shapes pred %s ratings %s' % (tuple(pred.shape), tuple(ratings.shape)))
    out = torch.empty(1, dtype=torch.float32, device=pred.device)
    g = torch.empty_like(p)
    ws = workspace('loss', lib.slb_loss_workspace_bytes(n), pred.device)
    rc = lib.slb_rating_loss(loss, _ptr(p), _ptr(r), n, _ptr(out), _ptr(g), _ptr(ws), ws.numel(), _stream())
    _lib.check(rc, 'rating_loss')
    return out.reshape(()), g.reshape(pred.shape)


@rating_loss.register_fake
def _(pred, ratings, loss):
    return pred.new_empty(()), torch.empty_like(pred)


def _rating_loss_setup(ctx, inputs, output):
    ctx.save_for_backward(output[1])


def _rating_loss_bwd(ctx, g_loss, g_grad):
    (d,) = ctx.saved_tensors
    return d * g_loss, None, None


rating_loss.register_autograd(_rating_loss_bwd, setup_context=_rating_loss_setup)


def rating_loss_op(kind: str, observed, predicted):
    """Scalar mean rating loss of ``predicted`` against ``observed`` (differentiable in
    ``predicted``)."""
    return rating_loss(predicted, observed, LOSS_KIND[kind])[0]


# ---------------------------------------------------------------------------
# Q1/Q2 sequence step                 spotlight/sequence/implicit.py:230-255
# ---------------------------------------------------------------------------

class _HostPtrArray(object):
    """Keeps the ctypes arrays of a slb_seq_step_args alive."""

    def __init__(self):
        self.keep = []

    def i32(self, values):
        arr = (ctypes.c_int32 * max(1, len(values)))(*[int(v) for v in values])
        self.keep.append(arr)
        return ctypes.cast(arr, ctypes.c_void_p)

    def ptrs(self, tensors):
        arr = (ctypes.c_void_p * max(1, len(tensors)))(*[t.data_ptr() for t in tensors])
        self.keep.append(arr)
        return ctypes.cast(arr, ctypes.c_void_p)


def seq_step_args(E, bias, seqs, negs, loss, n_neg, cnn=None, keep=None, lstm=None, mixture=None,
                  item_hash=None, num_items=None):
    """cnn: None (PoolNet) or dict(kernel_width, dilation, nonlinearity, residual, weights, biases);
    lstm: None or dict(w_ih, w_hh, b_ih, b_hh) (LSTMNet, nn.LSTM shapes);
    mixture: None or dict(num_mixtures, w, b) (MixtureLSTMNet's projection, with ``lstm``);
    item_hash: None or dict(seeds, padding_idx): ``E`` is a BloomEmbedding's hashed table and
    ``num_items`` the id space (the bias rows)."""
    keep = keep if keep is not None else _HostPtrArray()
    a = SeqStepArgs()
    a.batch, a.seq_len = int(seqs.shape[0]), int(seqs.shape[1])
    a.seqs = seqs.data_ptr()
    a.negs = negs.data_ptr() if negs is not None else None
    a.loss = LOSS_KIND[loss] if isinstance(loss, str) else int(loss)
    a.n_neg = int(n_neg)
    a.num_items, a.dim = int(E.shape[0]), int(E.shape[1])
    a.E, a.bias = E.data_ptr(), bias.data_ptr()
    if item_hash is not None:
        seeds = list(item_hash['seeds'])
        if not 1 <= len(seeds) <= 24:
            raise ValueError('item_hash: 1 to 24 seeds (got %d)' % len(seeds))
        a.num_items, a.item_rows, a.item_hashes = int(num_items), int(E.shape[0]), len(seeds)
        for k, s in enumerate(seeds):
            a.item_seeds[k] = int(s) & 0xFFFFFFFF
        a.item_padding_idx = int(item_hash['padding_idx'])
    if cnn is not None:
        a.n_layers = len(cnn['weights'])
        a.kernel_width = keep.i32(cnn['kernel_width'])
        a.dilation = keep.i32(cnn['dilation'])
        a.nonlinearity = 0 if cnn['nonlinearity'] == 'tanh' else 1
        a.residual = 1 if cnn['residual'] else 0
        a.conv_w = keep.ptrs(cnn['weights'])
        a.conv_b = keep.ptrs(cnn['biases'])
    if lstm is not None:
        a.lstm_w_ih, a.lstm_w_hh = lstm['w_ih'].data_ptr(), lstm['w_hh'].data_ptr()
        a.lstm_b_ih, a.lstm_b_hh = lstm['b_ih'].data_ptr(), lstm['b_hh'].data_ptr()
    if mixture is not None:
        a.num_mixtures = int(mixture['num_mixtures'])
        a.mix_w, a.mix_b = mixture['w'].data_ptr(), mixture['b'].data_ptr()
    return a, keep


_LSTM_KEYS = ('w_ih', 'w_hh', 'b_ih', 'b_hh')


def _lstm_params(lstm):
    if lstm is None:
        return None
    require_cuda(*[lstm[k] for k in _LSTM_KEYS])
    return {k: _f32c(lstm[k]) for k in _LSTM_KEYS}


def _mixture_params(mixture, lstm, D):
    """The Conv1d projection (2MD, D, 1) / (2MD,) as contiguous (2MD, D) / (2MD,) float32."""
    if mixture is None:
        return None
    if lstm is None:
        raise ValueError('mixture= needs lstm=: the mixture head sits on the LSTM representation')
    require_cuda(mixture['w'], mixture['b'])
    M = int(mixture['num_mixtures'])
    w = _f32c(mixture['w'])
    if w.numel() != 2 * M * D * D or w.shape[0] != 2 * M * D or mixture['b'].numel() != 2 * M * D:
        raise ValueError('mixture: projection of shape %s / %s does not map %d channels to 2 * %d * %d'
                         % (tuple(w.shape), tuple(mixture['b'].shape), D, M, D))
    return dict(num_mixtures=M, w=w.reshape(w.shape[0], -1), b=_f32c(mixture['b']))


def _seq_adam_args(a, fused, E, bias):
    """The lazy-exact Adam fields of slb_seq_step_args from ``fused`` (see seq_train_step)."""
    last_bias = fused.get('last_bias')
    tensors = [fused['state_E'], fused['state_bias'], fused['state2_E'], fused['state2_bias'], fused['last_E'],
               fused['sched']] + ([last_bias] if last_bias is not None else [])
    require_cuda(*tensors)
    for m, p in ((fused['state_E'], E), (fused['state2_E'], E), (fused['state_bias'], bias), (fused['state2_bias'], bias)):
        if m.shape != p.shape or m.dtype != torch.float32 or not m.is_contiguous():
            raise ValueError('seq_train_step: Adam moments must be contiguous float32 of the parameter shape')
    for last, p in ((fused['last_E'], E), (last_bias, bias)):
        if last is not None and (last.dtype != torch.int32 or last.shape != (p.shape[0],) or not last.is_contiguous()):
            raise ValueError('seq_train_step: Adam `last` must be contiguous int32 with one entry per row')
    if fused['sched'].numel() < 2 * (int(fused['step']) + 1):
        raise ValueError('seq_train_step: the Adam schedule does not reach step %d' % int(fused['step']))
    _adam_scalars(a, fused['beta1'], fused['beta2'], fused['sched'], fused['step'])
    a.state2_E, a.state2_bias = fused['state2_E'].data_ptr(), fused['state2_bias'].data_ptr()
    a.last_E = fused['last_E'].data_ptr()
    a.last_bias = last_bias.data_ptr() if last_bias is not None else None


def seq_train_step(E, bias, seqs, negs, loss, n_neg, cnn=None, want_scores=False, norm_count=None, fused=None,
                   lstm=None, mixture=None, item_hash=None):
    """Fused forward + backward of one sequence minibatch, dense gradients.

    Returns dict(loss, pos, neg, dE, dbias, dconv_w, dconv_b, dlstm).  ``fused`` = dict(kind, lr,
    weight_decay, eps, state_E, state_bias): the row-wise optimizer is applied to ``E`` / ``bias`` in
    place inside the step (no dense item-table gradient exists; ``dE`` / ``dbias`` are None).
    ``lstm`` = dict(w_ih, w_hh, b_ih, b_hh) selects the LSTMNet representation; ``dlstm`` then holds
    the gradients under the same keys.  ``mixture`` = dict(num_mixtures, w (2MD, D, 1), b (2MD,)), with
    ``lstm``, adds MixtureLSTMNet's projection and mixture-of-tastes scoring; ``dmix`` = dict(w, b)
    then holds the projection gradients in the shapes given.  ``item_hash`` = dict(seeds, padding_idx)
    makes ``E`` a ``BloomEmbedding``'s compressed (M, D) table: an item is the sum of its hashed rows,
    ``bias`` stays (num_items, 1), and ``dE`` is (M, D).

    Lazy-exact Adam (``optim.FusedAdam``): ``fused`` = dict(kind=OPT_ADAM, lr, weight_decay, eps, beta1,
    beta2, state_E / state_bias (exp_avg), state2_E / state2_bias (exp_avg_sq), last_E (int32, one entry
    per row of ``E``), last_bias (int32 (num_items,), hashed tables only; a plain table's bias shares
    last_E), sched (``FusedAdam.schedule``), step (this step, 1-based)).  The rows the minibatch
    references are first brought current through step - 1, then the rows with a gradient take step.
    """
    require_cuda(E, bias, seqs, negs)
    lib = _lib.load()
    E, bias = _f32c(E), _f32c(bias)
    seqs, negs = _i64c(seqs), _i64c(negs)
    B, S = seqs.shape
    dev = E.device
    if cnn is not None:
        cnn = dict(cnn)
        cnn['weights'] = [_f32c(w) for w in cnn['weights']]
        cnn['biases'] = [_f32c(b) for b in cnn['biases']]
    lstm = _lstm_params(lstm)
    mix = _mixture_params(mixture, lstm, int(E.shape[1]))
    a, keep = seq_step_args(E, bias, seqs, negs, loss, n_neg, cnn, lstm=lstm, mixture=mix, item_hash=item_hash,
                            num_items=bias.shape[0])
    out = dict(loss=torch.empty(1, dtype=torch.float32, device=dev), dE=None, dbias=None, dconv_w=[], dconv_b=[],
               dlstm=None, dmix=None)
    if fused is None:
        out['dE'], out['dbias'] = torch.zeros_like(E), torch.zeros_like(bias)
    a.loss_out = out['loss'].data_ptr()
    if want_scores:
        out['pos'] = torch.empty((B, S), dtype=torch.float32, device=dev)
        out['neg'] = torch.empty((n_neg * B, S), dtype=torch.float32, device=dev)
        a.pos_out, a.neg_out = out['pos'].data_ptr(), out['neg'].data_ptr()
    if fused is None:
        a.dE, a.dbias = out['dE'].data_ptr(), out['dbias'].data_ptr()
    else:
        a.opt, a.lr, a.weight_decay, a.eps = int(fused['kind']), float(fused['lr']), float(fused['weight_decay']), float(fused['eps'])
        if fused.get('state_E') is not None:
            a.state_E, a.state_bias = fused['state_E'].data_ptr(), fused['state_bias'].data_ptr()
        if a.opt == _lib.OPT_ADAM:
            _seq_adam_args(a, fused, E, bias)
    if norm_count is not None:
        a.norm_count = norm_count.data_ptr()
    if cnn is not None:
        out['dconv_w'] = [torch.zeros_like(w) for w in cnn['weights']]
        out['dconv_b'] = [torch.zeros_like(b) for b in cnn['biases']]
        a.dconv_w = keep.ptrs(out['dconv_w'])
        a.dconv_b = keep.ptrs(out['dconv_b'])
    if lstm is not None:
        out['dlstm'] = {k: torch.zeros_like(lstm[k]) for k in _LSTM_KEYS}
        a.dlstm_w_ih, a.dlstm_w_hh = out['dlstm']['w_ih'].data_ptr(), out['dlstm']['w_hh'].data_ptr()
        a.dlstm_b_ih, a.dlstm_b_hh = out['dlstm']['b_ih'].data_ptr(), out['dlstm']['b_hh'].data_ptr()
    if mix is not None:
        out['dmix'] = dict(w=torch.zeros(mixture['w'].shape, dtype=torch.float32, device=dev),
                           b=torch.zeros_like(mix['b']))
        a.dmix_w, a.dmix_b = out['dmix']['w'].data_ptr(), out['dmix']['b'].data_ptr()
    need = lib.slb_seq_step_workspace_bytes(ctypes.byref(a))
    # the zero-at-rest counters sit at offsets set by the key space: a hashed table has its own
    kind = 'seq%d' % a.num_items if item_hash is None else 'seqh%d_%d' % (a.num_items, a.item_rows)
    ws = workspace(kind, need, dev)
    a.workspace, a.workspace_bytes = ws.data_ptr(), ws.numel()
    _lib.check(lib.slb_seq_train_step(ctypes.byref(a), _stream()), 'seq_train_step')
    out['loss'] = out['loss'].reshape(())
    return out


def seq_representation(E, seqs, cnn=None, lstm=None, mixture=None):
    """(B, S+1, D) causal representations: entry t has seen items < t.  With ``mixture`` (see
    seq_train_step) the projection output, (B, S+1, 2MD), channel j*D + d of block j."""
    require_cuda(E, seqs)
    lib = _lib.load()
    E = _f32c(E)
    seqs = _i64c(seqs)
    B, S = seqs.shape
    if cnn is not None:
        cnn = dict(cnn)
        cnn['weights'] = [_f32c(w) for w in cnn['weights']]
        cnn['biases'] = [_f32c(b) for b in cnn['biases']]
    lstm = _lstm_params(lstm)
    mix = _mixture_params(mixture, lstm, int(E.shape[1]))
    dummy_bias = torch.zeros(1, dtype=torch.float32, device=E.device)
    a, keep = seq_step_args(E, dummy_bias, seqs, None, 0, 1, cnn, lstm=lstm, mixture=mix)
    width = E.shape[1] * (2 * mix['num_mixtures'] if mix is not None else 1)
    rep = torch.empty((B, S + 1, width), dtype=torch.float32, device=E.device)
    need = lib.slb_seq_step_workspace_bytes(ctypes.byref(a))
    ws = workspace('seq%d' % a.num_items, need, E.device)
    a.workspace, a.workspace_bytes = ws.data_ptr(), ws.numel()
    _lib.check(lib.slb_seq_representation(ctypes.byref(a), _ptr(rep), _stream()), 'seq_representation')
    return rep
