"""Secondary measurement (not bench.py's headline metric): the collective mrr_score and
precision_recall_score of ShardedImplicitFactorizationModel, scored on the item shards, against the
hand-off they replace -- gathered_net() followed by the single-GPU scorers on every rank.

Run under torchrun with one process per visible GPU, e.g.
    torchrun --nproc_per_node=$(nvidia-smi -L | wc -l) profiles/bench_eval_sharded.py --out result.json
(plain `python` runs world 1).  Shape of BASELINE config 2: 1M users x 100K items, D = 64, plain
tables, 100K test users with 10 test items each, a 5M-interaction train set excluded.  One more line
times a Bloom model: 1M item ids hashed to 200K rows, H = 4.

Before any timing the sharded outputs are compared with the hand-off's: equal at world 1; at larger
worlds the per-range GEMM may round a score differently from the full GEMM, and the number of users
whose result differs is reported.  Each arm is timed --rounds times after a warm-up call (host clock
around calls that end in a device synchronise: their results are NumPy arrays); medians are reported.
Rank 0 prints one JSON line with the GPU's name and power limit read in the same run; --out also
writes it there.  Multi-GPU scaling is "not measured" unless the run had several ranks."""
import argparse
import json
import os
import statistics
import sys
import tempfile
import time

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_seq_sharded import gpu_label   # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument('--users', type=int, default=1_000_000)
ap.add_argument('--items', type=int, default=100_000)
ap.add_argument('--dim', type=int, default=64)
ap.add_argument('--test-users', type=int, default=100_000)
ap.add_argument('--per-user', type=int, default=10)
ap.add_argument('--train', type=int, default=5_000_000)
ap.add_argument('--bloom-ids', type=int, default=1_000_000)
ap.add_argument('--bloom-rows', type=int, default=200_000)
ap.add_argument('--hashes', type=int, default=4)
ap.add_argument('--rounds', type=int, default=3)
ap.add_argument('--out', default=None)


def sets(a, num_items):
    from spotlight_b200.interactions import Interactions
    rs = np.random.RandomState(5)
    tu = np.repeat(rs.choice(a.users, a.test_users, replace=False), a.per_user)
    ti = rs.randint(0, num_items, len(tu))
    test = Interactions(tu.astype(np.int32), ti.astype(np.int32), num_users=a.users, num_items=num_items)
    train = Interactions(rs.randint(0, a.users, a.train).astype(np.int32),
                         rs.randint(0, num_items, a.train).astype(np.int32), num_users=a.users, num_items=num_items)
    return test, train


def wall_ms(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3, out


def handoff(model):
    """gathered_net() wrapped as the single-GPU scorers take a model."""
    import types
    net = model.gathered_net()
    return types.SimpleNamespace(_net=net, _optimizer=None, _num_items=model._num_items)


def differing_users(x, y):
    x, y = np.asarray(x), np.asarray(y)
    return int((x != y).reshape(len(x), -1).any(1).sum())


def measure(a, model, test, train):
    from spotlight_b200.evaluation import mrr_score, precision_recall_score
    ks = [1, 5, 10]
    arms = {
        'sharded_mrr': lambda: mrr_score(model, test, train),
        'sharded_precision_recall': lambda: precision_recall_score(model, test, train, k=ks),
        'gathered_mrr': lambda: mrr_score(handoff(model), test, train),
        'gathered_precision_recall': lambda: precision_recall_score(handoff(model), test, train, k=ks),
    }
    outs = {k: fn() for k, fn in arms.items()}                  # warm-up, and the outputs compared
    res = {'users_differing': {
        'mrr': differing_users(outs['sharded_mrr'], outs['gathered_mrr']),
        'precision': differing_users(outs['sharded_precision_recall'][0], outs['gathered_precision_recall'][0]),
        'recall': differing_users(outs['sharded_precision_recall'][1], outs['gathered_precision_recall'][1])},
        'users_scored': len(outs['sharded_mrr']), 'mean_mrr': float(np.mean(outs['sharded_mrr']))}
    if model.world == 1:
        assert all(v == 0 for v in res['users_differing'].values()), res
    else:
        assert all(v <= res['users_scored'] // 100 for v in res['users_differing'].values()), res
    times = {k: [] for k in arms}
    for _ in range(a.rounds):
        for k, fn in arms.items():                              # the arms alternate within each round
            times[k].append(wall_ms(fn)[0])
    res['ms_median'] = {k: statistics.median(v) for k, v in times.items()}
    res['ms_rounds'] = times
    return res


def main():
    a = ap.parse_args()
    from spotlight_b200.factorization.representations import BilinearNet
    from spotlight_b200.layers import BloomEmbedding
    from spotlight_b200.sharded import ShardedImplicitFactorizationModel
    rank, world = int(os.environ.get('RANK', 0)), int(os.environ.get('WORLD_SIZE', 1))
    dev = torch.device('cuda', int(os.environ.get('LOCAL_RANK', 0)))
    torch.cuda.set_device(dev)
    if 'RANK' in os.environ:
        dist.init_process_group('nccl', device_id=dev)
    else:
        store = 'file://' + os.path.join(tempfile.mkdtemp(prefix='bench_eval_sharded_'), 'store')
        dist.init_process_group('nccl', init_method=store, rank=0, world_size=1, device_id=dev)
    res = dict(gpu_label())
    res['world'] = world
    res['gpus_visible'] = torch.cuda.device_count()
    test, train = sets(a, a.items)
    torch.manual_seed(0)
    model = ShardedImplicitFactorizationModel(a.users, a.items, rank, world, dev, embedding_dim=a.dim,
                                              random_state=np.random.RandomState(1))
    res['plain'] = measure(a, model, test, train)
    res['plain']['config'] = ('users=%d items=%d D=%d test users=%d x %d items, train=%d'
                              % (a.users, a.items, a.dim, a.test_users, a.per_user, a.train))
    del model
    torch.manual_seed(0)
    net = BilinearNet(a.users, a.bloom_ids, a.dim, item_embedding_layer=BloomEmbedding(
        a.bloom_ids, a.dim, compression_ratio=a.bloom_rows / float(a.bloom_ids), num_hash_functions=a.hashes))
    model = ShardedImplicitFactorizationModel(a.users, a.bloom_ids, rank, world, dev, loss='hinge', representation=net,
                                              random_state=np.random.RandomState(1))
    test, train = sets(a, a.bloom_ids)
    res['bloom'] = measure(a, model, test, train)
    res['bloom']['config'] = ('users=%d item ids=%d hashed rows=%d H=%d D=%d test users=%d x %d items, train=%d'
                              % (a.users, a.bloom_ids, net.item_embeddings.compressed_num_embeddings, a.hashes,
                                 a.dim, a.test_users, a.per_user, a.train))
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
