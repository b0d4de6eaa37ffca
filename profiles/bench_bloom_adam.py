"""Implicit-feedback training with a Bloom item layer under Adam on one GPU: the in-place hashed
step with lazy-exact Adam against ``torch.optim.Adam`` on the dense ``bloom`` route.

Shape (BASELINE.json configs[3]): 1 M users (plain table), 50 M items hashed to 1 M rows
(compression ratio 0.02), H = 4, D = 64, hinge, B = 262 144; ``--items``, ``--ratio`` and
``--batch`` override it.  Both arms start from one initial state and run the same minibatches, in
alternating rounds, timed with CUDA events after warm-up:

* ``fused_adam``: ``ImplicitFactorizationModel._fit_epoch_bloom_fused``'s step under
  ``optim.fused_adam`` (``ops.mf_bloom_train_step_inplace`` with OPT_ADAM): rows and biases the
  minibatch reads are caught up, the touched ones take the step, no dense gradient anywhere;
* ``torch_adam``: the dense ``bloom`` route (``ops.fused_bloom_loss``: dense gradients of both
  tables and both id-indexed biases) and ``torch.optim.Adam`` over all of them.

Before timing, both arms run three steps on the same minibatches from the same state; the script
stops if a step's losses disagree, or if any of the four tables differs by more than 5 % of one
Adam step after the fused arm is flushed.  User, item and negative ids are drawn uniformly.  Prints one
JSON line with ms / step and interactions / s of each arm, the first losses, and the card's name and
power limit read in the same run; ``--out`` also writes it to a file.

    python profiles/bench_bloom_adam.py [--steps 10] [--warmup 2] [--rounds 3] [--out FILE]
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
from spotlight_b200.optim import FusedAdam  # noqa: E402

CHECK_STEPS = 3


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
    ap.add_argument('--out', default=None)
    lr, loss_name = 1e-3, 'hinge'
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_bloom_adam needs a CUDA device')
    dev = torch.device('cuda:0')
    U, I, D, B = args.users, args.items, args.dim, args.batch
    K = max(args.steps + args.warmup + 1, CHECK_STEPS)     # distinct minibatches
    torch.manual_seed(0)
    net = BilinearNet(U, I, D, user_embedding_layer=ScaledEmbedding(U, D),
                      item_embedding_layer=BloomEmbedding(I, D, compression_ratio=args.ratio,
                                                          num_hash_functions=args.hashes)).to(dev)
    g = torch.Generator(device=dev).manual_seed(1)
    users = torch.randint(0, U, (K, B), device=dev, generator=g)
    items = torch.randint(0, I, (K, B), device=dev, generator=g)
    negs = torch.randint(0, I, (K, B), device=dev, generator=g)

    # fused_adam: the in-place hashed step with lazy-exact Adam
    fnet = copy.deepcopy(net)
    spec = fnet.fused_spec()
    fparams = (spec['Wu'], spec['Wi'], fnet.user_biases.weight, fnet.item_biases.weight)
    fopt = FusedAdam(fnet.parameters(), lr=lr)
    fstates = [fopt.fused_states(p, own_last=True) for p in fparams]
    sched = fopt.schedule(4096, dev)
    hp = fopt.fused_hparams()
    tstep = [0]

    def fused(k):
        tstep[0] += 1
        return ops.mf_bloom_train_step_inplace(*fparams, users[k], items[k], negs[k], loss_name, 1,
                                               spec['user_seeds'], spec['item_seeds'], spec['user_pad'],
                                               spec['item_pad'], _lib.OPT_ADAM, lr, fstates, 0.0, hp['eps'],
                                               adam=dict(beta1=hp['beta1'], beta2=hp['beta2'], sched=sched,
                                                         step=tstep[0]))

    # torch_adam: the dense bloom route and torch.optim.Adam over every table
    dnet = copy.deepcopy(net)
    dspec = dnet.fused_spec()
    dopt = torch.optim.Adam(dnet.parameters(), lr=lr)

    def dense(k):
        dopt.zero_grad()
        loss = ops.fused_bloom_loss(dspec['Wu'], dspec['Wi'], dnet.user_biases.weight, dnet.item_biases.weight,
                                    users[k], items[k], negs[k], loss_name, 1, dspec)
        loss.backward()
        dopt.step()
        return loss.detach()

    # before timing: three steps of both arms on the same minibatches from the same state, then the
    # fused arm flushed (exact: it only replays pending gradient-free steps) and all four tables
    # compared, so a wrong catch-up or apply stops the script, not only a wrong forward
    first = None
    for k in range(CHECK_STEPS):
        lf, ld = float(fused(k)), float(dense(k))
        if abs(lf - ld) > 1e-5 * max(1.0, abs(ld)):
            raise SystemExit('step %d losses disagree: %r' % (k + 1, (lf, ld)))
        first = first or dict(fused_adam=lf, torch_adam=ld)
    fopt.advance(tstep[0])
    fopt.flush()
    table_err = {}
    with torch.no_grad():
        for nm, p, q in zip(('Wu', 'Wi', 'bu', 'bi'), fparams,
                            (dspec['Wu'], dspec['Wi'], dnet.user_biases.weight, dnet.item_biases.weight)):
            err = (p - q).abs().max().item()
            table_err[nm] = err
            if err > 0.05 * lr + 2e-6 * q.abs().max().item():
                raise SystemExit('%s differs after %d steps by %.3e' % (nm, CHECK_STEPS, err))

    def timed(fn):
        for k in range(args.warmup):
            fn(1 + k)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for k in range(args.steps):
            fn(1 + args.warmup + k)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / args.steps

    res = {'fused_adam_ms': [], 'torch_adam_ms': []}
    for _ in range(args.rounds):
        res['fused_adam_ms'].append(timed(fused))
        res['torch_adam_ms'].append(timed(dense))
    name, power = _card()
    out = dict(shape=dict(users=U, items=I, rows=spec['Wi'].shape[0], hashes=args.hashes, dim=D, batch=B),
               loss=loss_name, optimizer='adam', lr=lr, ids='uniform', card=name, power_limit=power,
               first_step_loss=first, checked_steps=CHECK_STEPS, table_max_abs_err=table_err, **res)
    for k in ('fused_adam', 'torch_adam'):
        out[k + '_interactions_per_s'] = [B / (ms * 1e-3) for ms in res[k + '_ms']]
    out['speedup'] = min(res['torch_adam_ms']) / min(res['fused_adam_ms'])
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
