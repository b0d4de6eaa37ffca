"""Secondary measurement (not bench.py's headline metric): sharded sequence training with row-wise
lazy-exact Adam (optimizer_func=fused_adam) at bench_seq_sharded.py's shape: 1M items, dim 128,
S = 200, pointwise loss, PoolNet and LSTMNet, minibatches of --batches.

Runs at world 1 and, when N > 1 GPUs are visible, at world N (one process per GPU, NCCL).  For each
net and batch, three arms on the same minibatches, alternated --rounds times, each round timing
--steps steps with CUDA events after two warm-up steps (ms/step is the median round):
  * the estimator's step with fused_adam (owner catch-up, exchange, fused step on the row cache,
    owner Adam, replicated Adam);
  * the estimator's step with its default row-wise Adagrad;
  * ImplicitSequenceModel(optimizer_func=fused_adam) on one GPU (world 1 only).
The first global losses of the two Adam arms must agree (relative 1e-5) before anything is timed.
Then the owner update alone on the rows one step hands a world-1 owner (the distinct ids of the
minibatch): slb_shard_rows_adam and slb_shard_rows_adam_catch_up against slb_shard_rows_adagrad.
Prints one JSON line per case and a final summary with the GPU's name and power limit read in the
same run; --out also writes the summary there."""
import json
import os
import sys

import numpy as np
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_seq_sharded import ROOT, ap, gpu_label, minibatches, timed   # noqa: E402,F401

ADAM = dict(lr=1e-3, weight_decay=1e-6)


def run_case(a, rank, world, dev, rep, B):
    from spotlight_b200.interactions import SequenceInteractions
    from spotlight_b200.optim import fused_adam
    from spotlight_b200.sequence.implicit import ImplicitSequenceModel
    from spotlight_b200.sharded import ShardedImplicitSequenceModel, _rank_slice
    batches = minibatches(a, B, dev)
    lo, hi = _rank_slice(B, rank, world)

    def estimator(opt):
        est = ShardedImplicitSequenceModel(a.items, rank, world, dev, loss='pointwise', representation=rep,
                                           embedding_dim=a.dim, batch_size=B, learning_rate=0.05,
                                           random_state=np.random.RandomState(42), optimizer_func=opt)

        def step(k):
            s, n = batches[k]
            return est.seq.step(s[lo:hi], n[lo:hi], 'pointwise')
        return step

    arms = {'sharded_fused_adam': estimator(fused_adam(**ADAM)), 'sharded_adagrad': estimator(None)}
    if rank == 0 and world == 1:
        single = ImplicitSequenceModel(loss='pointwise', representation=rep, embedding_dim=a.dim, batch_size=B,
                                       use_cuda=True, random_state=np.random.RandomState(42),
                                       optimizer_func=fused_adam(**ADAM))
        single._initialize(SequenceInteractions(np.ones((1, a.seq), dtype=np.int64), num_items=a.items))
        assert single._route() == 'fused'

        def single_step(k):
            s, n = batches[k]
            single._optimizer.zero_grad()
            loss = single._fused_step(s, n, 1)
            single._optimizer.step()
            return loss
        arms['single_gpu_fused_adam'] = single_step
    first = {name: float(fn(0)) for name, fn in arms.items()}
    res = {'world': world, 'net': rep, 'batch': B, 'first_losses': first}
    if 'single_gpu_fused_adam' in first:
        l_est, l_one = first['sharded_fused_adam'], first['single_gpu_fused_adam']
        if abs(l_est - l_one) > 1e-5 * abs(l_one):
            raise SystemExit('first losses disagree: %r vs %r' % (l_est, l_one))
    for fn in arms.values():
        fn(1)
    rounds = {name: [] for name in arms}
    for _ in range(a.rounds):
        for name, fn in arms.items():
            dist.barrier()
            rounds[name].append(timed(fn, 2, 2 + a.steps))
    for name in arms:
        res[name + '_ms_per_step'] = float(np.median(rounds[name]))
        res[name + '_ms_rounds'] = rounds[name]
    return res


def owner_update_case(a, dev, B):
    """The owner updates alone, on the distinct ids of one minibatch (world 1: every row comes home
    to the one owner).  Each Adam call is a new step, so every row is a step behind when it
    arrives: the catch-up finds nothing to replay and the step applies one Adam step per row."""
    import types
    from spotlight_b200.optim import FusedAdam
    from spotlight_b200.sharded import GpuBackend
    s, n = minibatches(a, B, dev)[0]
    ids = torch.unique(torch.cat([s.reshape(-1), n.reshape(-1)]))
    R, D, rows = ids.numel(), a.dim, a.items
    g = torch.randn(R, D, device=dev) * 1e-3
    gb = torch.randn(R, device=dev) * 1e-3
    z = lambda *shape: torch.zeros(*shape, device=dev)        # noqa: E731
    st = types.SimpleNamespace(Wi=torch.randn(rows, D, device=dev), sWi=z(rows, D), bi=z(rows), sbi=z(rows),
                               lr=0.05, eps=1e-10, mWi=z(rows, D), vWi=z(rows, D), mbi=z(rows), vbi=z(rows),
                               last=torch.zeros(rows, dtype=torch.int32, device=dev),
                               opt=FusedAdam([z(1)], **ADAM))
    be = GpuBackend(dev)
    calls = {'rows_adagrad': lambda k: be.owner_update(st, ids, g, gb),
             'rows_adam': lambda k: be.owner_adam_update(st, ids, g, gb, k + 1),
             'rows_adam_catch_up': lambda k: be.owner_adam_catch_up(st, ids, k + 1)}
    for fn in calls.values():
        fn(0)
    times = {name: [] for name in calls}
    k = 1
    for _ in range(a.rounds):
        for name, fn in calls.items():
            times[name].append(timed(fn, k, k + 20))
        k += 20
    out = {'owner_update': True, 'batch': B, 'rows_received': R, 'shard_rows': rows, 'dim': D}
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
        for rep in a.nets.split(','):
            for B in [int(x) for x in a.batches.split(',')]:
                r = run_case(a, rank, world, dev, rep, B)
                torch.cuda.empty_cache()
                if rank == 0:
                    print(json.dumps(r), flush=True)
                    out.append(r)
        if rank == 0 and world == 1:
            for B in [int(x) for x in a.batches.split(',')]:
                r = owner_update_case(a, dev, B)
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
    summary = dict(gpu_label(), config='ImplicitSequenceModel pointwise items=%d D=%d S=%d fused_adam %s'
                   % (a.items, a.dim, a.seq, ADAM), gpus_visible=n, steps=a.steps, rounds=a.rounds, results=results,
                   not_measured=[] if n > 1 else ['world > 1: one GPU visible'])
    print(json.dumps(summary), flush=True)
    if a.out:
        with open(a.out, 'w') as f:
            json.dump(summary, f, indent=1)
