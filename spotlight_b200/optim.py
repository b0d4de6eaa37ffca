"""Row-wise optimizers fused into the training step (SURVEY §8f row f1).

The reference's default ``optim.Adam`` (spotlight/factorization/implicit.py:
143-148) sweeps every embedding row each minibatch -- 72 % of its step at
1M x 100K x 64.  SGD and Adagrad change a row only when its gradient is
non-zero, so applying them to the touched rows alone is *exactly* the dense
update (no weight decay / momentum); here that update runs in
``mf_apply_kernel`` right after the gradient kernel, never materialising a
dense gradient.

Both classes are ordinary ``torch.optim`` optimizers (usable with any module
via ``.step()``); ``ImplicitFactorizationModel.fit`` recognises them through
``fused_kind`` and switches to the on-device epoch pipeline.

Use as ``optimizer_func``::

    model = ImplicitFactorizationModel(loss='bpr', use_cuda=True,
                                       optimizer_func=fused_adagrad(lr=0.05))
"""

import torch

from spotlight_b200 import _lib


class FusedSGD(torch.optim.SGD):
    """Plain SGD (no momentum).  ``weight_decay``: on the fused pipelines it is applied to the
    rows a minibatch updates only (see ``FusedAdagrad``)."""

    fused_kind = _lib.OPT_SGD

    def __init__(self, params, lr=1e-2, weight_decay=0.0):
        super(FusedSGD, self).__init__(params, lr=lr, momentum=0.0, weight_decay=weight_decay)

    def fused_hparams(self):
        g = self.param_groups[0]
        return dict(lr=float(g['lr']), weight_decay=float(g['weight_decay']), eps=0.0)

    def fused_state(self, param):
        return None


class FusedAdagrad(torch.optim.Adagrad):
    """Adagrad with ``lr_decay = 0`` and ``initial_accumulator_value = 0``
    (torch defaults).  State lives in ``self.state[p]['sum']`` exactly as in
    ``torch.optim.Adagrad`` so training can continue with either.

    ``weight_decay``: on the fused pipelines it is added (as ``wd * w``) to the gradient of the
    rows a minibatch updates only, in every element of such a row; torch's dense Adagrad decays
    every row on every step.  A row is updated when one of its terms has a non-zero score
    gradient (in a sequence step also when its embedding gradient is non-zero, through the
    item's input role), even if its own embedding gradient is exactly zero; a bias is updated
    with its row, so the user bias of a bpr / hinge interaction (gp + gn = 0) is decayed too.  With
    ``weight_decay = 0`` (the default) this is the dense update; with ``weight_decay > 0`` rows
    outside the minibatch are not decayed."""

    fused_kind = _lib.OPT_ADAGRAD

    def __init__(self, params, lr=1e-2, weight_decay=0.0, eps=1e-10):
        super(FusedAdagrad, self).__init__(params, lr=lr, lr_decay=0.0,
                                           weight_decay=weight_decay,
                                           initial_accumulator_value=0.0, eps=eps)

    def fused_hparams(self):
        g = self.param_groups[0]
        return dict(lr=float(g['lr']), weight_decay=float(g['weight_decay']), eps=float(g['eps']))

    def fused_state(self, param):
        return self.state[param]['sum']


class FusedAdam(torch.optim.Optimizer):
    """Row-wise *lazy-exact* Adam: the reference's default optimizer
    (``optim.Adam(params, weight_decay=l2, lr=learning_rate)``,
    spotlight/factorization/implicit.py:143-148) at O(batch) per step.

    Dense Adam moves every row every step (a row without a gradient still moves, its first
    moment decays).  Here a row is brought up to date when it is next touched: the steps it
    missed are replayed for it element by element with torch's own recurrence
    (csrc/mf_adam.cuh), then the real step is applied.  ``flush()`` replays what is pending
    for every row; ``ImplicitFactorizationModel.fit`` calls it before returning, so the
    parameters the caller sees are those of dense Adam (up to fp32 rounding of identical
    formulas).  State (``exp_avg``, ``exp_avg_sq``, ``step``) is kept in ``self.state`` under
    torch's names plus a per-row ``last`` step index.

    Any module: the tables a fused step updates lazily (the factorization models' tables, a
    sequence model's item table and bias) are registered through ``fused_states`` and flushed;
    every other parameter (convolutions, LSTM, projection) takes ordinary dense Adam in
    ``step()``, which on the fused routes runs after the kernel with the same step count.

    Hyperparameters may change between steps (``param_groups[0]``, by hand or through a
    ``torch.optim.lr_scheduler``): dense Adam took the steps a row missed with the values of their
    time, so before the first use of new values every pending step is flushed with the values it
    was taken under, and the schedule is rebuilt.  One O(table) flush per change.
    """

    fused_kind = _lib.OPT_ADAM

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0):
        defaults = dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay)
        super(FusedAdam, self).__init__(params, defaults)
        self._t = 0                      # optimizer steps taken (torch's state['step'])
        self._sched = None
        self._hp = None                  # the hyperparameters the lazy state was advanced with

    # torch.optim.Optimizer pickles only defaults / state / param_groups: keep the step count so
    # that a pickled model resumes fit() with the right bias corrections, and the hyperparameters
    # of its pending steps
    def __getstate__(self):
        st = super(FusedAdam, self).__getstate__()
        st['_t'] = self._t
        st['_hp'] = self._hp
        return st

    def __setstate__(self, state):
        state = dict(state)
        self._t = state.pop('_t', 0)
        self._hp = state.pop('_hp', None)
        self._sched = None
        super(FusedAdam, self).__setstate__(state)

    # ---- state ----------------------------------------------------------------
    def fused_hparams(self):
        g = self.param_groups[0]
        return dict(lr=float(g['lr']), weight_decay=float(g['weight_decay']), eps=float(g['eps']),
                    beta1=float(g['betas'][0]), beta2=float(g['betas'][1]))

    def _moments(self, param):
        st = self.state[param]
        if 'exp_avg' not in st:
            st['exp_avg'] = torch.zeros_like(param)
            st['exp_avg_sq'] = torch.zeros_like(param)
        if 'last' not in st:
            st['last'] = torch.full((param.shape[0],), self._t, dtype=torch.int32, device=param.device)
        return st['exp_avg'], st['exp_avg_sq'], st['last']

    def fused_states(self, param, own_last=False):
        """``(exp_avg, exp_avg_sq, last)`` of a table a fused step updates lazily; registers it for
        ``flush()``.  By default the table is one half of an (embedding, bias) pair that shares the
        embedding's ``last`` (the factorization models, a plain sequence item table); ``own_last``:
        a table flushed on its own with its own ``last`` (a hashed item table, an id-indexed bias)."""
        states = self._moments(param)
        self.state[param]['lazy'] = 'own' if own_last else 'pair'
        return states

    def _current_hparams(self):
        """``fused_hparams()``, after the lazy state has caught up with any change of them: when
        they differ from those the pending steps were taken under, every lazy table is flushed
        with the recorded values first and the schedule is dropped.  ``schedule()``, ``flush()``
        and ``step()`` all start here."""
        hp = self.fused_hparams()
        if self._hp is not None and hp != self._hp:
            self._flush(self._hp)
            self._sched = None
        self._hp = hp
        return hp

    def schedule(self, upto, device):
        """Device table of the per-step scalars lr / (1 - beta1^t), sqrt(1 - beta2^t), t <= upto
        (computed in double, as torch's Python does)."""
        return self._schedule(self._current_hparams(), upto, device)

    def _schedule(self, hp, upto, device):
        import numpy as np
        if self._sched is None or self._sched.shape[0] < 2 * (upto + 1) or self._sched.device != device:
            cap = max(4096, 2 * upto)
            t = np.arange(cap + 1, dtype=np.float64)
            tab = np.empty((cap + 1, 2), dtype=np.float64)
            with np.errstate(divide='ignore'):
                tab[:, 0] = hp['lr'] / (1.0 - hp['beta1'] ** t)
            tab[:, 1] = np.sqrt(1.0 - hp['beta2'] ** t)
            tab[0] = 0.0
            self._sched = torch.from_numpy(tab.astype(np.float32).reshape(-1)).to(device)
        return self._sched

    @property
    def steps_taken(self):
        return self._t

    def advance(self, k):
        """Record ``k`` fused steps taken by the epoch pipeline."""
        self._t += int(k)
        for st in self.state.values():
            st['step'] = self._t

    def _lazy(self, kind):
        return [p for g in self.param_groups for p in g['params'] if self.state.get(p, {}).get('lazy') == kind]

    def flush(self):
        """Replay the pending (gradient-free) steps of every row of the lazily updated tables (those
        registered through ``fused_states``); every other parameter is always current."""
        self._flush(self._current_hparams())

    def _flush(self, hp):
        """``flush()`` with the hyperparameters ``hp``."""
        from spotlight_b200 import ops
        if self._t == 0:
            return
        lib = _lib.load()
        scalars = (hp['beta1'], hp['beta2'], 1.0 - hp['beta1'], 1.0 - hp['beta2'], hp['eps'], hp['weight_decay'],
                   ops._stream())
        params = self._lazy('pair')
        # tables come in (embedding (rows, D), bias (rows, 1)) pairs sharing `last`: the k-th
        # embedding table pairs with the k-th bias table (BilinearNet's parameter order)
        emb = [p for p in params if p.dim() == 2 and p.shape[1] > 1]
        bias = [p for p in params if p.dim() == 2 and p.shape[1] == 1]
        if len(emb) != len(bias) or any(W.shape[0] != b.shape[0] for W, b in zip(emb, bias)):
            raise RuntimeError('FusedAdam.flush: expected (embedding, bias) table pairs')
        for W, b in zip(emb, bias):
            if not W.is_cuda:
                continue        # CPU tensors only ever see the dense step() below, which leaves every row current
            rows = W.shape[0]
            m, v, last = self.fused_states(W)
            bm, bv, _ = self.fused_states(b)
            sched = self._schedule(hp, self._t, W.device)
            with torch.no_grad():
                _lib.check(lib.slb_adam_flush(ops._ptr(W), ops._ptr(m), ops._ptr(v), ops._ptr(b), ops._ptr(bm),
                                              ops._ptr(bv), ops._ptr(last), rows, W.shape[1], ops._ptr(sched),
                                              self._t, *scalars), 'adam_flush')
        for p in self._lazy('own'):
            if not p.is_cuda:
                continue
            m, v, last = self._moments(p)
            sched = self._schedule(hp, self._t, p.device)
            with torch.no_grad():
                _lib.check(lib.slb_adam_flush_table(ops._ptr(p), ops._ptr(m), ops._ptr(v), ops._ptr(last),
                                                    p.shape[0], p[0].numel(), ops._ptr(sched), self._t, *scalars),
                           'adam_flush_table')

    def step(self, closure=None):
        """One ordinary Adam step (step count t = steps taken + 1) on every parameter that has a
        ``.grad``.  A lazily updated table that has no ``.grad`` (a fused sequence step already
        applied step t to it in place) is left alone.  When a lazily updated table does carry a
        ``.grad`` (the dense fallback for callers that drive the optimizer themselves), every lazy
        table is flushed first, so the dense step finds all rows current.  Every stepped parameter
        keeps a ``last`` (= t after the step) so that a table a fused path registers later starts
        current.  Sparse gradients are rejected, as torch.optim.Adam rejects them."""
        loss = closure() if closure is not None else None
        params = [p for g in self.param_groups for p in g['params'] if p.grad is not None]
        hp = self._current_hparams()
        if any(self.state.get(p, {}).get('lazy') for p in params):
            self._flush(hp)
        self._t += 1
        t = self._t
        ss = hp['lr'] / (1.0 - hp['beta1'] ** t)
        bc2s = (1.0 - hp['beta2'] ** t) ** 0.5
        lasts = []
        with torch.no_grad():
            for p in params:
                if p.grad.is_sparse:
                    raise RuntimeError('FusedAdam does not support sparse gradients (as torch.optim.Adam): '
                                       'construct the model with sparse=False')
                m, v, last = self._moments(p)
                grad = p.grad if hp['weight_decay'] == 0 else p.grad.add(p, alpha=hp['weight_decay'])
                m.lerp_(grad, 1 - hp['beta1'])
                v.mul_(hp['beta2']).addcmul_(grad, grad, value=1 - hp['beta2'])
                p.addcdiv_(m, (v.sqrt() / bc2s).add_(hp['eps']), value=-ss)
                lasts.append(last)
            if lasts:                  # every stepped parameter is current for t: two multi-tensor launches
                torch._foreach_zero_(lasts)
                torch._foreach_add_(lasts, t)
        for st in self.state.values():
            st['step'] = t
        return loss


class _Factory(object):
    """Picklable ``optimizer_func`` (models are saved whole with ``torch.save``)."""

    def __init__(self, cls, **kwargs):
        self.cls = cls
        self.kwargs = kwargs

    def __call__(self, params):
        return self.cls(params, **self.kwargs)


def fused_sgd(lr=1e-2, weight_decay=0.0):
    """``optimizer_func`` factory for :class:`FusedSGD`."""
    return _Factory(FusedSGD, lr=lr, weight_decay=weight_decay)


def fused_adam(lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0):
    """``optimizer_func`` factory for :class:`FusedAdam` (row-wise lazy-exact Adam)."""
    return _Factory(FusedAdam, lr=lr, betas=betas, eps=eps, weight_decay=weight_decay)


def fused_adagrad(lr=1e-2, weight_decay=0.0, eps=1e-10):
    """``optimizer_func`` factory for :class:`FusedAdagrad`."""
    return _Factory(FusedAdagrad, lr=lr, weight_decay=weight_decay, eps=eps)
