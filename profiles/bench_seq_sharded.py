"""Secondary measurement (not bench.py's headline metric): sequence training on N GPUs through
ShardedImplicitSequenceModel at BASELINE.json configs[4]'s shape: 1M items, dim 128, S = 200,
pointwise loss, PoolNet and LSTMNet, minibatches of --batches.

Runs at world 1 and, when N > 1 GPUs are visible, at world N (one process per GPU, NCCL).  For each
net and batch:
  * the estimator's step (ShardedSeq.step on this rank's contiguous slice of each global minibatch:
    bucketing, row all-to-alls, fused step on the row cache, owner update, replicated-parameter
    all-reduce) against ImplicitSequenceModel(optimizer_func=fused_adagrad) on the same minibatches,
    both from one seed; the first global losses must agree (relative 1e-5) before anything is timed.
    The single-GPU arm is timed at world 1 only.  Arms alternate --rounds times; each round times
    --steps steps with CUDA events after two warm-up steps; ms/step is the median round.
  * the owner update alone on the rows one step hands a world-1 owner (the distinct ids of the
    minibatch, as received): slb_shard_rows_adagrad against the dense route it replaces
    (embedding_backward into a (rows, D) gradient + slb_adagrad_dense over the shard), alternated.
Prints one JSON line per case and a final summary with the GPU's name and power limit read in the
same run; --out also writes the summary there."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

ap = argparse.ArgumentParser()
ap.add_argument('--items', type=int, default=1_000_000)
ap.add_argument('--dim', type=int, default=128)
ap.add_argument('--seq', type=int, default=200)
ap.add_argument('--steps', type=int, default=10)
ap.add_argument('--rounds', type=int, default=3)
ap.add_argument('--nets', default='pooling,lstm')
ap.add_argument('--batches', default='256,1024')
ap.add_argument('--out', default=None)


def gpu_label():
    try:
        pl = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', '0'],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = 'unknown'
    return {'gpu': torch.cuda.get_device_name(0), 'nvidia_smi': pl or 'unknown'}


def minibatches(a, B, dev):
    from spotlight_b200.sampling import sample_items
    g = torch.Generator(device=dev)
    g.manual_seed(B)
    n = (a.steps + 3) * B
    seqs = torch.randint(1, a.items, (n, a.seq), device=dev, generator=g)
    pad = torch.randint(0, a.seq, (n,), device=dev, generator=g)
    seqs[torch.arange(a.seq, device=dev)[None, :] < pad[:, None] // 4] = 0
    negs = sample_items(a.items, (n, a.seq), random_state=np.random.RandomState(B), device=dev)
    return [(seqs[k * B:(k + 1) * B], negs[k * B:(k + 1) * B]) for k in range(a.steps + 3)]


def timed(fn, k0, k1):
    """ms per call of fn(k) for k in [k0, k1), CUDA events."""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for k in range(k0, k1):
        fn(k)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / (k1 - k0)


def run_case(a, rank, world, dev, rep, B):
    from spotlight_b200.interactions import SequenceInteractions
    from spotlight_b200.optim import fused_adagrad
    from spotlight_b200.sequence.implicit import ImplicitSequenceModel
    from spotlight_b200.sharded import ShardedImplicitSequenceModel, _rank_slice
    batches = minibatches(a, B, dev)
    est = ShardedImplicitSequenceModel(a.items, rank, world, dev, loss='pointwise', representation=rep,
                                       embedding_dim=a.dim, batch_size=B, learning_rate=0.05,
                                       random_state=np.random.RandomState(42))
    lo, hi = _rank_slice(B, rank, world)

    def est_step(k):
        s, n = batches[k]
        return est.seq.step(s[lo:hi], n[lo:hi], 'pointwise')

    single = None
    if rank == 0:
        single = ImplicitSequenceModel(loss='pointwise', representation=rep, embedding_dim=a.dim, batch_size=B,
                                       use_cuda=True, random_state=np.random.RandomState(42),
                                       optimizer_func=fused_adagrad(lr=0.05))
        single._initialize(SequenceInteractions(np.ones((1, a.seq), dtype=np.int64), num_items=a.items))
        assert single._route() == 'fused'

    def single_step(k):
        s, n = batches[k]
        single._optimizer.zero_grad()
        loss = single._fused_step(s, n, 1)
        single._optimizer.step()
        return loss

    l_est = float(est_step(0))
    res = {'world': world, 'net': rep, 'batch': B}
    if rank == 0:
        l_one = float(single_step(0))
        res.update(first_loss_estimator=l_est, first_loss_single=l_one)
        if abs(l_est - l_one) > 1e-5 * abs(l_one):
            raise SystemExit('first losses disagree: %r vs %r' % (l_est, l_one))
        if world > 1:
            del single
            single = None
            torch.cuda.empty_cache()
    est_step(1)
    if single is not None:
        single_step(1)
    est_ms, one_ms = [], []
    for _ in range(a.rounds):
        dist.barrier()
        est_ms.append(timed(est_step, 2, 2 + a.steps))
        if single is not None:
            one_ms.append(timed(single_step, 2, 2 + a.steps))
    res['estimator_ms_per_step'] = float(np.median(est_ms))
    res['estimator_ms_rounds'] = est_ms
    if one_ms:
        res['single_gpu_fused_adagrad_ms_per_step'] = float(np.median(one_ms))
        res['single_ms_rounds'] = one_ms
    return res


def owner_update_case(a, dev, B):
    """The owner update alone, on the distinct ids of one minibatch (world 1: every row comes home
    to the one owner)."""
    import types
    from spotlight_b200 import _lib, ops
    from spotlight_b200.sharded import GpuBackend
    s, n = minibatches(a, B, dev)[0]
    ids = torch.unique(torch.cat([s.reshape(-1), n.reshape(-1)]))
    R, D, rows = ids.numel(), a.dim, a.items
    g = torch.randn(R, D, device=dev) * 1e-3
    gb = torch.randn(R, device=dev) * 1e-3
    st = types.SimpleNamespace(Wi=torch.randn(rows, D, device=dev), sWi=torch.zeros(rows, D, device=dev),
                               bi=torch.zeros(rows, device=dev), sbi=torch.zeros(rows, device=dev), lr=0.05, eps=1e-10)
    be, lib = GpuBackend(dev), _lib.load()

    def new(_):
        be.owner_update(st, ids, g, gb)

    def old(_):
        dW = ops.embedding_backward(g, ids, [], rows, -1)
        db = ops.embedding_backward(gb.reshape(-1, 1), ids, [], rows, -1)
        for W, S, G in ((st.Wi, st.sWi, dW), (st.bi, st.sbi, db.reshape(-1))):
            _lib.check(lib.slb_adagrad_dense(ops._ptr(W), ops._ptr(S), ops._ptr(G), W.numel(), st.lr, st.eps,
                                             ops._stream()), 'adagrad_dense')

    new(0)
    old(0)
    t_new, t_old = [], []
    for _ in range(a.rounds):
        t_new.append(timed(new, 0, 20))
        t_old.append(timed(old, 0, 20))
    return {'owner_update': True, 'batch': B, 'rows_received': R, 'shard_rows': rows, 'dim': D,
            'rows_adagrad_ms': float(np.median(t_new)), 'dense_backward_plus_adagrad_ms': float(np.median(t_old)),
            'rows_adagrad_rounds': t_new, 'dense_rounds': t_old}


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
    port = 29600 + (os.getpid() + world) % 1000
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
    summary = dict(gpu_label(), config='ImplicitSequenceModel pointwise items=%d D=%d S=%d' % (a.items, a.dim, a.seq),
                   gpus_visible=n, steps=a.steps, rounds=a.rounds, results=results,
                   not_measured=[] if n > 1 else ['world > 1: one GPU visible'])
    print(json.dumps(summary), flush=True)
    if a.out:
        with open(a.out, 'w') as f:
            json.dump(summary, f, indent=1)
