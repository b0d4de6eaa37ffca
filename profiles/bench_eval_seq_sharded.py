"""Secondary measurement (not bench.py's headline metric): the collective sequence_mrr_score of
ShardedImplicitSequenceModel, scored on the item shards, against the hand-off it replaces --
gathered_net() followed by the single-GPU scorer on every rank.

Run under torchrun with one process per visible GPU, e.g.
    torchrun --nproc_per_node=$(nvidia-smi -L | wc -l) profiles/bench_eval_seq_sharded.py --out result.json
(plain `python` runs world 1).  Shape: 1M items, D = 128, 4096 test sequences of length 200 (left
padding of random length), PoolNet, LSTMNet and MixtureLSTMNet (M = 4) at their initial weights, blocks
of 256 sequences (the scorers' default).

Before any timing the sharded output is compared with the hand-off's: equal at world 1; at larger
worlds the per-range GEMM may round a dot-head score differently from the full GEMM, and the number of
sequences whose result differs is reported.  The arms alternate within each of --rounds rounds after a
warm-up call (host clock around calls that end in a device synchronise: their results are NumPy
arrays); medians are reported.  Rank 0 prints one JSON line with the GPU's name and power limit read in
the same run; --out also writes it there.  Multi-GPU scaling is "not measured" unless the run had
several ranks."""
import argparse
import json
import os
import statistics
import sys
import tempfile
import time
import types

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_seq_sharded import gpu_label   # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument('--items', type=int, default=1_000_000)
ap.add_argument('--dim', type=int, default=128)
ap.add_argument('--seq', type=int, default=200)
ap.add_argument('--test', type=int, default=4096)
ap.add_argument('--mixtures', type=int, default=4)
ap.add_argument('--nets', default='pooling,lstm,mixture')
ap.add_argument('--rounds', type=int, default=3)
ap.add_argument('--out', default=None)


def test_set(a):
    from spotlight_b200.interactions import SequenceInteractions
    rs = np.random.RandomState(5)
    seqs = rs.randint(1, a.items, (a.test, a.seq)).astype(np.int64)
    pad = rs.randint(0, a.seq - 1, a.test)
    seqs[np.arange(a.seq) < pad[:, None]] = 0
    return SequenceInteractions(seqs, num_items=a.items)


def wall_ms(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3, out


def handoff(model):
    """gathered_net() wrapped as the single-GPU scorers take a model."""
    return types.SimpleNamespace(_net=model.gathered_net(), _optimizer=None, _num_items=model._num_items)


def measure(a, model, test):
    from spotlight_b200.evaluation import sequence_mrr_score
    arms = {'sharded_mrr': lambda: sequence_mrr_score(model, test),
            'gathered_mrr': lambda: sequence_mrr_score(handoff(model), test)}
    outs = {k: fn() for k, fn in arms.items()}                  # warm-up, and the outputs compared
    res = {'sequences_differing': int((outs['sharded_mrr'] != outs['gathered_mrr']).sum()),
           'sequences_scored': len(outs['sharded_mrr']), 'mean_mrr': float(np.mean(outs['sharded_mrr']))}
    if model.world == 1:
        assert res['sequences_differing'] == 0, res
    times = {k: [] for k in arms}
    for _ in range(a.rounds):
        for k, fn in arms.items():                              # the arms alternate within each round
            times[k].append(wall_ms(fn)[0])
    res['ms_median'] = {k: statistics.median(v) for k, v in times.items()}
    res['ms_rounds'] = times
    return res


def main():
    a = ap.parse_args()
    from spotlight_b200.sequence.representations import LSTMNet, MixtureLSTMNet, PoolNet
    from spotlight_b200.sharded import ShardedImplicitSequenceModel
    rank, world = int(os.environ.get('RANK', 0)), int(os.environ.get('WORLD_SIZE', 1))
    dev = torch.device('cuda', int(os.environ.get('LOCAL_RANK', 0)))
    torch.cuda.set_device(dev)
    if 'RANK' in os.environ:
        dist.init_process_group('nccl', device_id=dev)
    else:
        store = 'file://' + os.path.join(tempfile.mkdtemp(prefix='bench_eval_seq_sharded_'), 'store')
        dist.init_process_group('nccl', init_method=store, rank=0, world_size=1, device_id=dev)
    res = dict(gpu_label())
    res['world'] = world
    res['gpus_visible'] = torch.cuda.device_count()
    res['config'] = 'items=%d D=%d test sequences=%d S=%d block=256' % (a.items, a.dim, a.test, a.seq)
    test = test_set(a)
    builders = {'pooling': lambda: PoolNet(a.items, a.dim), 'lstm': lambda: LSTMNet(a.items, a.dim),
                'mixture': lambda: MixtureLSTMNet(a.items, a.dim, num_mixtures=a.mixtures)}
    for name in a.nets.split(','):
        torch.manual_seed(0)
        model = ShardedImplicitSequenceModel(a.items, rank, world, dev, representation=builders[name](),
                                             embedding_dim=a.dim, random_state=np.random.RandomState(1))
        res[name] = measure(a, model, test)
        del model
        torch.cuda.empty_cache()
    res['multi_gpu'] = 'not measured' if world < 2 else 'world %d' % world
    if rank == 0:
        line = json.dumps(res)
        print(line)
        if a.out:
            with open(a.out, 'w') as f:
                f.write(line + '\n')
    dist.destroy_process_group()


if __name__ == '__main__':
    main()
