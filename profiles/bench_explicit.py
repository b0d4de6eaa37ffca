"""Explicit-feedback MF step throughput on one GPU.

At the headline shape (1M users x 100K items x 64, B = 524 288, device-resident ids) it times the
regression step with fused Adagrad (the model's epoch route) and, alternately in the same process,
the BPR step with fused Adagrad, with CUDA events over `--steps` steps each.  Both run the planned
two-kernel step (csrc/mf_v2.cuh; the regression step in its one-term mode).

It also times the user kernel alone (`slb_mf_train_step_phases`, phase 2, CUDA events around
each launch) and divides its algorithmic bytes by that time.  Per interaction (R = 4·D bytes, one
user row per interaction as in a uniform batch), the one-term user kernel reads U[u] and Q[i], two
biases and the 16-byte member record, and writes U[u] and one g: 3R + 28 bytes (796 B at D = 64).
The BPR user kernel reads one more item row and bias and writes one more g: 4R + 36 (1060 B, the
figure bench.py reports).  Optimizer state rows are not counted, as in bench.py.

With `--ref-ml100k` it times the unmodified reference's CPU `fit()` (`oracle/_ref`, placed there
by `build()`) at the MovieLens-100K shape (943 users, 1682 items, 100 000 ratings, D = 32,
batch 256, regression, default Adam) on one epoch.

Prints one JSON line with the rates, the card's name and power limit.

    python profiles/bench_explicit.py [--steps 50] [--warmup 5] [--rounds 3]
"""

import argparse
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from spotlight_b200 import _lib, ops  # noqa: E402
from spotlight_b200.sampling import sample_items  # noqa: E402


def _card():
    try:
        out = subprocess.check_output(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                                      text=True).strip().split('\n')[0]
        return [x.strip() for x in out.split(',')]
    except (OSError, subprocess.CalledProcessError):
        return [torch.cuda.get_device_name(), 'unknown']


def reference_ml100k():
    """One epoch of the unmodified reference's explicit fit() on the host CPU (oracle/_ref)."""
    import time
    ref = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'oracle', '_ref')
    if not os.path.isdir(os.path.join(ref, 'spotlight')):
        raise SystemExit('oracle/_ref is missing: run build() first')
    sys.path.insert(0, ref)
    from spotlight.factorization.explicit import ExplicitFactorizationModel
    from spotlight.interactions import Interactions
    rs = np.random.RandomState(0)
    n, U, I = 100_000, 943, 1682
    inter = Interactions(rs.randint(0, U, n).astype(np.int32), rs.randint(0, I, n).astype(np.int32),
                         ratings=rs.randint(1, 6, n).astype(np.float32), num_users=U, num_items=I)
    model = ExplicitFactorizationModel(loss='regression', embedding_dim=32, n_iter=1, batch_size=256,
                                       random_state=np.random.RandomState(1))
    t0 = time.perf_counter()
    model.fit(inter)
    dt = time.perf_counter() - t0
    return dict(seconds_per_epoch=dt, interactions_per_s=n / dt, threads=torch.get_num_threads())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=50)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--users', type=int, default=1_000_000)
    ap.add_argument('--items', type=int, default=100_000)
    ap.add_argument('--dim', type=int, default=64)
    ap.add_argument('--batch', type=int, default=524_288)
    ap.add_argument('--ref-ml100k', action='store_true')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_explicit needs a CUDA device')
    dev = torch.device('cuda:0')
    g = torch.Generator(device=dev).manual_seed(0)
    U, I, D, B, K = args.users, args.items, args.dim, args.batch, args.steps
    params = [torch.randn(U, D, device=dev, generator=g) / 8, torch.randn(I, D, device=dev, generator=g) / 8,
              torch.zeros(U, 1, device=dev), torch.zeros(I, 1, device=dev)]
    states = [torch.zeros_like(p) for p in params]
    users = torch.randint(0, U, (K, B), device=dev, generator=g)
    items = torch.randint(0, I, (K, B), device=dev, generator=g)
    ratings = torch.randint(1, 6, (K, B), device=dev, generator=g).float()
    negs = sample_items(I, K * B, random_state=np.random.RandomState(1), device=dev).view(K, B)

    def explicit(k):
        ops.mf_train_step_inplace(*params, users[k], items[k], None, 'regression', _lib.OPT_ADAGRAD, 1e-3, states,
                                  ratings=ratings[k])

    def bpr(k):
        ops.mf_train_step_inplace(*params, users[k], items[k], negs[k], 'bpr', _lib.OPT_ADAGRAD, 1e-3, states)

    def timed(fn):
        for k in range(args.warmup):
            fn(k % K)
        torch.cuda.synchronize()
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for k in range(K):
            fn(k)
        t1.record()
        torch.cuda.synchronize()
        return t0.elapsed_time(t1) / K

    def user_kernel_ms(loss, neg, rating):
        """Mean CUDA-event time of the user-kernel phase of the planned step."""
        lib = _lib.load()
        ms = []
        for k in range(K):
            a = ops.mf_step_args(*params, users[k], items[k], neg[k] if neg is not None else None, loss, 1,
                                 ratings=rating[k] if rating is not None else None)
            loss_out = torch.empty(1, device=dev)
            a.loss_out = loss_out.data_ptr()
            a.grad_mode = _lib.GRAD_COMPACT
            a.opt, a.lr, a.eps = _lib.OPT_ADAGRAD, 1e-3, 1e-10
            a.state_Wu, a.state_Wi, a.state_bu, a.state_bi = [t.data_ptr() for t in states]
            fneed = lib.slb_mf_fused_workspace_bytes(B, U, I, D)
            fws = ops.workspace('mfv2_%d_%d_%d' % (U, I, D), fneed, dev)
            a.fused_workspace, a.fused_workspace_bytes = fws.data_ptr(), fws.numel()
            need = lib.slb_mf_step_workspace_bytes(B, 1, a.loss, U, I)
            ws = ops.workspace('mf%d_%d' % (U, I), need, dev)
            a.workspace, a.workspace_bytes = ws.data_ptr(), ws.numel()
            st = ops._stream()
            _lib.check(lib.slb_mf_train_step_phases(ctypes.byref(a), 1, st), 'plan')
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            _lib.check(lib.slb_mf_train_step_phases(ctypes.byref(a), 2, st), 'user')
            e1.record()
            _lib.check(lib.slb_mf_train_step_phases(ctypes.byref(a), 4, st), 'item')
            torch.cuda.synchronize()
            if k >= 1:
                ms.append(e0.elapsed_time(e1))
        return sum(ms) / len(ms)

    res = {'explicit_regression_ms': [], 'bpr_planned_ms': []}
    for _ in range(args.rounds):
        res['explicit_regression_ms'].append(timed(explicit))
        res['bpr_planned_ms'].append(timed(bpr))
    name, power = _card()
    out = dict(shape=[U, I, D, B], optimizer='fused adagrad', card=name, power_limit=power, **res)
    for k in ('explicit_regression', 'bpr_planned'):
        out[k + '_interactions_per_s'] = [B / (ms * 1e-3) for ms in res[k + '_ms']]
    R = 4 * D
    for k, loss, neg, rating, per in (('explicit_regression', 'regression', None, ratings, 3 * R + 28),
                                      ('bpr_planned', 'bpr', negs, None, 4 * R + 36)):
        t = user_kernel_ms(loss, neg, rating)
        out[k + '_user_kernel'] = dict(ms=t, algorithmic_bytes_per_interaction=per,
                                       achieved_gbs=per * B / (t * 1e-3) / 1e9)
    if args.ref_ml100k:
        out['reference_cpu_ml100k'] = reference_ml100k()
    print(json.dumps(out))


if __name__ == '__main__':
    main()
