"""Secondary measurement (not bench.py's headline metric): sharded factorization training with row-wise
lazy-exact Adam (optimizer_func=fused_adam) at config 2's shape: 1M users x 100K items x dim 64, BPR.

Runs at world 1 and, when N > 1 GPUs are visible, at world N (one process per GPU, NCCL).  For each
minibatch size -- by default one below and one above the dense-exchange threshold (2 B / world >=
items), so the a2a and the dense exchange are both measured under exchange='auto' -- three arms on
the same minibatches, alternated --rounds times, each round timing --steps steps with CUDA events
after two warm-up steps (ms/step is the median round):
  * ShardedMF.step with fused_adam (owner catch-up or whole-shard catch-up, users-only Adam step,
    owner Adam or dense Adam on the shard);
  * ShardedMF.step with the default row-wise Adagrad;
  * ImplicitFactorizationModel(optimizer_func=fused_adam) on one GPU (world 1 only), one step of its
    epoch pipeline.
The first global losses of the two Adam arms must agree (relative 1e-5) before anything is timed.
Then adaptive hinge at config 3's shape (10M users x 1M items x dim 128, 5 negatives, --ada-batch),
the same three arms through ShardedMF.step_adaptive: under fused_adam the scored user rows are caught
up and the whole user shard takes slb_adam_dense from its dense gradient, under Adagrad the dense
Adagrad pass; the first losses of the Adam arms must agree to 1e-4 (the sharded route scores with
mf_scores, the single-GPU step with its fused forward).  Then the owner-side dense sweep alone on the
100K-row item shard: slb_adam_dense against slb_adagrad_dense.  Prints one JSON line per case and a final summary with the GPU's name and power
limit read in the same run; --out also writes the summary there."""
import argparse
import json
import os
import sys

import numpy as np
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_seq_sharded import ROOT, gpu_label, timed   # noqa: E402,F401

ADAM = dict(lr=1e-3, weight_decay=1e-6)

ap = argparse.ArgumentParser()
ap.add_argument('--users', type=int, default=1_000_000)
ap.add_argument('--items', type=int, default=100_000)
ap.add_argument('--dim', type=int, default=64)
ap.add_argument('--steps', type=int, default=20)
ap.add_argument('--rounds', type=int, default=3)
ap.add_argument('--batches', default='4096,65536')
ap.add_argument('--ada-users', type=int, default=10_000_000)
ap.add_argument('--ada-items', type=int, default=1_000_000)
ap.add_argument('--ada-dim', type=int, default=128)
ap.add_argument('--ada-batch', type=int, default=4096)
ap.add_argument('--ada-neg', type=int, default=5)
ap.add_argument('--ada-steps', type=int, default=10)
ap.add_argument('--out', default=None)


def minibatches(a, B, dev, n=64, n_neg=1):
    g = torch.Generator(device=dev)
    g.manual_seed(B)
    return [tuple(torch.randint(0, hi, (m,), generator=g, device=dev)
                  for hi, m in ((a.users, B), (a.items, B), (a.items, B * n_neg))) for _ in range(n)]


def params(a, dev):
    g = torch.Generator(device=dev)
    g.manual_seed(7)
    D = a.dim
    return [torch.randn(a.users, D, generator=g, device=dev) / D, torch.randn(a.items, D, generator=g, device=dev) / D,
            torch.zeros(a.users, 1, device=dev), torch.zeros(a.items, 1, device=dev)]


def run_case(a, rank, world, dev, B, loss='bpr', n_neg=1, steps=None):
    from spotlight_b200.factorization.implicit import ImplicitFactorizationModel
    from spotlight_b200.interactions import Interactions
    from spotlight_b200.optim import fused_adam
    from spotlight_b200.sharded import ShardedImplicitFactorizationModel
    steps = steps or a.steps
    batches = minibatches(a, B, dev, 16 if n_neg > 1 else 64, n_neg)
    init = params(a, dev)

    def estimator(opt):
        est = ShardedImplicitFactorizationModel(a.users, a.items, rank, world, dev, loss=loss, embedding_dim=a.dim,
                                                batch_size=B, learning_rate=0.05, random_state=np.random.RandomState(42),
                                                exchange='auto', init=init, optimizer_func=opt,
                                                num_negative_samples=n_neg)
        plan = est.plan

        def step(k):
            u, i, j = batches[k % len(batches)]
            mine = torch.nonzero(plan.user_owner(u) == rank).reshape(-1)
            if loss == 'adaptive_hinge':
                block = j.reshape(B, n_neg)[mine].reshape(-1)
                return est.mf.step_adaptive(u[mine], i[mine], block, mine, u, n_neg)
            return est.mf.step(u[mine], i[mine], j[mine], loss, B, 'auto')
        return step, est

    adam_step, est = estimator(fused_adam(**ADAM))
    arms = {'sharded_fused_adam': adam_step, 'sharded_adagrad': estimator(None)[0]}
    dense = est.mf._dense_exchange_pays(B // world)
    if rank == 0 and world == 1:
        single = ImplicitFactorizationModel(loss=loss, embedding_dim=a.dim, batch_size=B, use_cuda=True,
                                            random_state=np.random.RandomState(42), optimizer_func=fused_adam(**ADAM),
                                            num_negative_samples=n_neg)
        single._initialize(Interactions(np.zeros(1, np.int32), np.zeros(1, np.int32), num_users=a.users,
                                        num_items=a.items))
        net = single._net
        with torch.no_grad():
            for prm, val in zip((net.user_embeddings.weight, net.item_embeddings.weight, net.user_biases.weight,
                                 net.item_biases.weight), init):
                prm.copy_(val.reshape(prm.shape))

        def single_step(k):
            u, i, j = batches[k % len(batches)]
            return single._fit_epoch_pipeline(u, i, j, sync=False)
        arms['single_gpu_fused_adam'] = single_step
    del init
    first = {name: float(fn(0)) for name, fn in arms.items()}
    res = {'world': world, 'loss': loss, 'users': a.users, 'items': a.items, 'dim': a.dim, 'batch': B,
           'exchange': 'score routing' if loss == 'adaptive_hinge' else ('dense' if dense else 'a2a'),
           'first_losses': first}
    if 'single_gpu_fused_adam' in first:
        l_est, l_one = first['sharded_fused_adam'], first['single_gpu_fused_adam']
        if abs(l_est - l_one) > (1e-4 if loss == 'adaptive_hinge' else 1e-5) * abs(l_one):
            raise SystemExit('first losses disagree: %r vs %r' % (l_est, l_one))
    for fn in arms.values():
        fn(1)
    rounds = {name: [] for name in arms}
    k = 2
    for _ in range(a.rounds):
        for name, fn in arms.items():
            dist.barrier()
            rounds[name].append(timed(fn, k, k + steps))
        k += steps
    for name in arms:
        res[name + '_ms_per_step'] = float(np.median(rounds[name]))
        res[name + '_ms_rounds'] = rounds[name]
    return res


def owner_sweep_case(a, dev):
    """The owner-side dense update alone on the item shard (world 1: all items rows): dense Adam
    (each call a new step, every row one step behind, so the catch-up replays nothing) against
    Adagrad."""
    import types
    from spotlight_b200.optim import FusedAdam
    from spotlight_b200.sharded import GpuBackend
    rows, D = a.items, a.dim
    z = lambda *shape: torch.zeros(*shape, device=dev)        # noqa: E731
    g, gb = torch.randn(rows, D, device=dev) * 1e-3, torch.randn(rows, device=dev) * 1e-3
    st = types.SimpleNamespace(Wi=torch.randn(rows, D, device=dev), sWi=z(rows, D), bi=z(rows), sbi=z(rows),
                               mWi=z(rows, D), vWi=z(rows, D), mbi=z(rows), vbi=z(rows),
                               last=torch.zeros(rows, dtype=torch.int32, device=dev), opt=FusedAdam([z(1)], **ADAM))
    be = GpuBackend(dev)
    calls = {'adagrad_dense': lambda k: (be.adagrad_dense(st.Wi, st.sWi, g, 0.05, 1e-10),
                                         be.adagrad_dense(st.bi, st.sbi, gb, 0.05, 1e-10)),
             'adam_dense': lambda k: be.adam_dense(st, False, g, gb, k + 1)}
    for fn in calls.values():
        fn(0)
    times = {name: [] for name in calls}
    k = 1
    for _ in range(a.rounds):
        for name, fn in calls.items():
            times[name].append(timed(fn, k, k + 50))
        k += 50
    out = {'owner_sweep': True, 'shard_rows': rows, 'dim': D}
    for name in calls:
        out[name + '_ms'] = float(np.median(times[name]))
        out[name + '_rounds'] = times[name]
    return out


def worker(rank, world, port, a, q):
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    torch.cuda.set_device(rank)
    dev = torch.device('cuda', rank)
    dist.init_process_group('nccl', rank=rank, world_size=world, device_id=dev)
    out = []
    try:
        for B in [int(x) for x in a.batches.split(',')]:
            r = run_case(a, rank, world, dev, B)
            torch.cuda.empty_cache()
            if rank == 0:
                print(json.dumps(r), flush=True)
                out.append(r)
        ada = argparse.Namespace(users=a.ada_users, items=a.ada_items, dim=a.ada_dim, steps=a.ada_steps,
                                 rounds=a.rounds)
        r = run_case(ada, rank, world, dev, a.ada_batch, 'adaptive_hinge', a.ada_neg)
        torch.cuda.empty_cache()
        if rank == 0:
            print(json.dumps(r), flush=True)
            out.append(r)
        if rank == 0 and world == 1:
            r = owner_sweep_case(a, dev)
            print(json.dumps(r), flush=True)
            out.append(r)
        q.put((rank, out, None))
    except BaseException:
        import traceback
        q.put((rank, None, traceback.format_exc()))
    finally:
        dist.destroy_process_group()


def run_world(a, world):
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = 29700 + (os.getpid() + world) % 1000
    procs = [ctx.Process(target=worker, args=(r, world, port, a, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = {}
    for _ in range(world):
        rank, out, err = q.get(timeout=3600)
        if err is not None:
            for p in procs:
                p.terminate()
            raise SystemExit('rank %d failed:\n%s' % (rank, err))
        res[rank] = out
    for p in procs:
        p.join(timeout=120)
    return res[0]


if __name__ == '__main__':
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('needs a CUDA device')
    n = torch.cuda.device_count()
    results = run_world(a, 1)
    if n > 1:
        results += run_world(a, n)
    summary = dict(gpu_label(), config='ImplicitFactorizationModel bpr users=%d items=%d D=%d; adaptive_hinge '
                   'users=%d items=%d D=%d n_neg=%d; fused_adam %s'
                   % (a.users, a.items, a.dim, a.ada_users, a.ada_items, a.ada_dim, a.ada_neg, ADAM), gpus_visible=n,
                   steps=a.steps, ada_steps=a.ada_steps, rounds=a.rounds, results=results,
                   not_measured=[] if n > 1 else ['world > 1: one GPU visible'])
    print(json.dumps(summary), flush=True)
    if a.out:
        with open(a.out, 'w') as f:
            json.dump(summary, f, indent=1)
