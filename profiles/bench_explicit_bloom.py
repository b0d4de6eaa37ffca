"""Explicit-feedback training with a Bloom item layer on one GPU: route ``bloom`` against
``generic``.

Shape (BASELINE.json configs[3] with ratings): 1 M users (plain table), 50 M items hashed to
1 M rows (compression ratio 0.02), H = 4, D = 64, regression, B = 262 144; ``--items``,
``--ratio`` and ``--batch`` override it.  Both routes start from one initial state and run the
same minibatches, in alternating rounds, timed with CUDA events after warm-up:

* ``bloom``: ``ExplicitFactorizationModel._fit_epoch_bloom_fused``'s step, the fused hashed-table
  step with fused Adagrad applied in place (``ops.mf_bloom_train_step_inplace``);
* ``generic``: the reference's loop body on the same net, autograd through the Bloom gather and
  ``torch.optim.Adagrad`` (a dense gradient and update of every table).

Prints one JSON line: ms / step and interactions / s of each route, both routes' loss on the
first minibatch from the same state, and the card's name and power limit read in the same run.

    python profiles/bench_explicit_bloom.py [--steps 10] [--warmup 2] [--rounds 3]
"""

import argparse
import copy
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from spotlight_b200 import _lib, ops  # noqa: E402
from spotlight_b200.factorization.representations import BilinearNet  # noqa: E402
from spotlight_b200.layers import BloomEmbedding, ScaledEmbedding  # noqa: E402
from spotlight_b200.losses import regression_loss  # noqa: E402


def _card():
    try:
        out = subprocess.check_output(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                                      text=True).strip().split('\n')[0]
        return [x.strip() for x in out.split(',')]
    except (OSError, subprocess.CalledProcessError):
        return [torch.cuda.get_device_name(), 'unknown']


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--users', type=int, default=1_000_000)
    ap.add_argument('--items', type=int, default=50_000_000)
    ap.add_argument('--ratio', type=float, default=0.02)
    ap.add_argument('--hashes', type=int, default=4)
    ap.add_argument('--dim', type=int, default=64)
    ap.add_argument('--batch', type=int, default=262_144)
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--rounds', type=int, default=3)
    lr = 0.05
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_explicit_bloom needs a CUDA device')
    dev = torch.device('cuda:0')
    U, I, D, B, K = args.users, args.items, args.dim, args.batch, args.steps
    torch.manual_seed(0)
    net = BilinearNet(U, I, D, user_embedding_layer=ScaledEmbedding(U, D),
                      item_embedding_layer=BloomEmbedding(I, D, compression_ratio=args.ratio,
                                                          num_hash_functions=args.hashes)).to(dev)
    g = torch.Generator(device=dev).manual_seed(1)
    users = torch.randint(0, U, (K, B), device=dev, generator=g)
    items = torch.randint(0, I, (K, B), device=dev, generator=g)
    ratings = torch.randint(1, 6, (K, B), device=dev, generator=g).float()

    # bloom route: the fused hashed-table step with Adagrad in place
    bnet = copy.deepcopy(net)
    spec = bnet.fused_spec()
    bparams = (spec['Wu'], spec['Wi'], bnet.user_biases.weight, bnet.item_biases.weight)
    bstates = [torch.zeros_like(p) for p in bparams]

    def bloom(k):
        return ops.mf_bloom_train_step_inplace(*bparams, users[k], items[k], None, 'regression', 1,
                                               spec['user_seeds'], spec['item_seeds'], spec['user_pad'],
                                               spec['item_pad'], _lib.OPT_ADAGRAD, lr, bstates,
                                               ratings=ratings[k])

    # generic route: autograd through the Bloom gather, dense torch.optim.Adagrad
    gnet = copy.deepcopy(net)
    gopt = torch.optim.Adagrad(gnet.parameters(), lr=lr)

    def generic(k):
        gopt.zero_grad()
        loss = regression_loss(ratings[k], gnet(users[k], items[k]))
        loss.backward()
        gopt.step()
        return loss.detach()

    first = dict(bloom=float(bloom(0)), generic=float(generic(0)))   # same state, same minibatch

    def timed(fn):
        for k in range(args.warmup):
            fn(k % K)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for k in range(K):
            fn(k)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / K

    res = {'bloom_ms': [], 'generic_ms': []}
    for _ in range(args.rounds):
        res['bloom_ms'].append(timed(bloom))
        res['generic_ms'].append(timed(generic))
    name, power = _card()
    out = dict(shape=dict(users=U, items=I, rows=spec['Wi'].shape[0], hashes=args.hashes, dim=D, batch=B),
               loss='regression', optimizer='adagrad', card=name, power_limit=power, first_step_loss=first, **res)
    for k in ('bloom', 'generic'):
        out[k + '_interactions_per_s'] = [B / (ms * 1e-3) for ms in res[k + '_ms']]
    out['speedup'] = min(res['generic_ms']) / min(res['bloom_ms'])
    print(json.dumps(out))


if __name__ == '__main__':
    main()
