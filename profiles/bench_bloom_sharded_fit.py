"""Secondary measurement (not bench.py's headline metric): ShardedImplicitFactorizationModel.fit() on a
BilinearNet with a BloomEmbedding item layer at BASELINE config 4's shape -- 1M users, 50M item ids
hashed to 1M rows, D = 64, H = 4, hinge, B = 131 072 per rank -- with fused_adam and with Adagrad.

World 1 in this process.  Several GPUs are needed for the multi-GPU numbers; with one visible they are
reported as "not measured".  Each arm fits --steps minibatches (one epoch) after a warm-up fit, and
the time per step is the fit's wall time (ending in a device synchronise) over its steps: shuffle,
negative stream and the final Adam flush included.

Then the local step alone, in the same process, alternating --rounds rounds: the dense-user form
(dense dWu over the whole user shard, then slb_adagrad_dense over it and the sparse user-bias update)
against the users-only mode (user rows and biases updated in place at O(batch)), both Adagrad, on the
same minibatches.  Prints one JSON line with the GPU's name and power limit read in the same run;
--out also writes it there."""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_seq_sharded import ROOT, gpu_label, timed   # noqa: E402,F401

ap = argparse.ArgumentParser()
ap.add_argument('--users', type=int, default=1_000_000)
ap.add_argument('--items', type=int, default=50_000_000)
ap.add_argument('--ratio', type=float, default=0.02)          # 50M ids -> 1M hashed rows
ap.add_argument('--dim', type=int, default=64)
ap.add_argument('--hashes', type=int, default=4)
ap.add_argument('--batch', type=int, default=131072)
ap.add_argument('--steps', type=int, default=20)
ap.add_argument('--rounds', type=int, default=5)
ap.add_argument('--out', default=None)


def bloom_net(a):
    from spotlight_b200.factorization.representations import BilinearNet
    from spotlight_b200.layers import BloomEmbedding
    torch.manual_seed(0)
    return BilinearNet(a.users, a.items, a.dim,
                       item_embedding_layer=BloomEmbedding(a.items, a.dim, compression_ratio=a.ratio,
                                                           num_hash_functions=a.hashes))


def fit_ms(a, dev, optimizer_func, users, items):
    """ms per step of a one-epoch fit() after a warm-up fit of the same model."""
    import torch.distributed as dist
    from spotlight_b200.interactions import Interactions
    from spotlight_b200.sharded import ShardedImplicitFactorizationModel
    if not dist.is_initialized():
        import tempfile
        store = 'file://' + os.path.join(tempfile.mkdtemp(prefix='bench_bloom_'), 'store')
        dist.init_process_group('nccl', init_method=store, rank=0, world_size=1, device_id=dev)
    model = ShardedImplicitFactorizationModel(a.users, a.items, 0, 1, dev, loss='hinge', n_iter=1,
                                              batch_size=a.batch, random_state=np.random.RandomState(1),
                                              optimizer_func=optimizer_func, representation=bloom_net(a))
    inter = Interactions(users, items, num_users=a.users, num_items=a.items)
    model.fit(inter)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    model.fit(inter)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / a.steps, model.epoch_losses[-1]


def local_step_ms(a, dev):
    """(dense-user ms, users-only ms) of the local hashed step, median of alternated rounds."""
    from spotlight_b200 import ops
    from spotlight_b200.layers import SEEDS
    from spotlight_b200.sharded import BloomShardState, GpuBackend, ShardPlan
    plan = ShardPlan(a.users, a.items, 1)
    M = int(a.ratio * a.items)
    st = BloomShardState(plan, 0, a.dim, dev, a.items, M, a.hashes)
    be = GpuBackend(dev)
    seeds = [int(x) for x in SEEDS[:a.hashes]]
    g = torch.Generator(device=dev)
    g.manual_seed(5)
    K = 8
    batches = [(torch.randint(0, a.users, (a.batch,), device=dev, generator=g),
                torch.randint(1, a.items, (a.batch,), device=dev, generator=g),
                torch.randint(0, a.items, (a.batch,), device=dev, generator=g)) for _ in range(K)]

    def dense_user(k):
        u, i, n = batches[k % K]
        _, dWu, _, (iu, gu), _ = ops.mf_bloom_step_pairs(st.Wu, st.Wi, st.bu2, st.bi2, u, i, n, 'hinge', seeds, 0,
                                                         norm_batch=a.batch)
        be.adagrad_dense(st.Wu, st.sWu, dWu, st.lr, st.eps)
        be.bias_sparse_adagrad(iu, gu, st.bu, st.sbu, st.lr, st.eps)

    def users_only(k):
        u, i, n = batches[k % K]
        be.bloom_local_step(st, st.Wi, u, i, n, 'hinge', a.batch)

    for fn in (dense_user, users_only):
        fn(0)
    torch.cuda.synchronize()
    dense, uo = [], []
    for _ in range(a.rounds):
        dense.append(timed(dense_user, 0, a.steps))
        uo.append(timed(users_only, 0, a.steps))
    return statistics.median(dense), statistics.median(uo), dense, uo


def main():
    a = ap.parse_args()
    from spotlight_b200 import optim
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    rs = np.random.RandomState(3)
    n = a.steps * a.batch
    users = rs.randint(0, a.users, n).astype(np.int32)
    items = rs.randint(1, a.items, n).astype(np.int32)
    res = dict(gpu_label())
    res['config'] = ('ShardedImplicitFactorizationModel(representation=BilinearNet + BloomEmbedding) hinge users=%d '
                     'item ids=%d hashed rows=%d D=%d H=%d B=%d per rank' % (a.users, a.items, int(a.ratio * a.items),
                                                                           a.dim, a.hashes, a.batch))
    res['gpus_visible'] = torch.cuda.device_count()
    adam_ms, adam_loss = fit_ms(a, dev, optim.fused_adam(lr=1e-3, weight_decay=1e-6), users, items)
    ada_ms, ada_loss = fit_ms(a, dev, None, users, items)
    res['world1_fit_ms_per_step'] = {'fused_adam': adam_ms, 'adagrad': ada_ms}
    res['world1_epoch_loss'] = {'fused_adam': adam_loss, 'adagrad': ada_loss}
    d, u, dr, ur = local_step_ms(a, dev)
    res['local_step_ms'] = {'dense_user_adagrad': d, 'users_only_adagrad': u,
                            'rounds': {'dense_user_adagrad': dr, 'users_only_adagrad': ur}}
    res['multi_gpu'] = 'not measured' if torch.cuda.device_count() < 2 else 'run with torchrun (not in this process)'
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, 'w') as f:
            f.write(line + '\n')
    import torch.distributed as dist
    if dist.is_initialized():
        dist.destroy_process_group()


if __name__ == '__main__':
    main()
