"""Secondary measurement (not bench.py's headline metric): sequence models trained with Adam, the
reference's default optimizer, at BASELINE.json configs[4]'s shape: 1M items, dim 128, S = 200,
pointwise loss.

For each representation of --arms (pool, cnn_k3, lstm, mixture with 4 tastes on a plain item
table; bloom_pool, bloom_lstm on a BloomEmbedding item layer, ratio 0.2, 4 hashes) and each batch
of --batches it times ImplicitSequenceModel's step on two arms from one initial state and the same
minibatches.  Plain tables: optim.fused_adam (lazy-exact Adam inside the fused step, then
optimizer.step() on the net's own parameters) against torch.optim.Adam on the same fused route
(a dense (items, D) gradient and a sweep over the table and both moments).  Bloom tables:
fused_adam on the fused_hashed route against torch.optim.Adam on the generic route.  Before
timing, the first two steps' losses of both arms are compared (relative difference at most 1e-5,
else the script stops): the first compares the forward on one state, the second the update.  The arms alternate --rounds times; each round times --steps
steps with CUDA events after two warm-up steps.  Prints ms/step (median round), positions/s and
the GPU's name and power limit read in the same run."""
import argparse, json, os, subprocess, sys
import numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from spotlight_b200.sampling import sample_items

ap = argparse.ArgumentParser()
ap.add_argument('--items', type=int, default=1_000_000); ap.add_argument('--ratio', type=float, default=0.2)
ap.add_argument('--hashes', type=int, default=4); ap.add_argument('--dim', type=int, default=128)
ap.add_argument('--seq', type=int, default=200); ap.add_argument('--steps', type=int, default=10)
ap.add_argument('--arms', default='pool,cnn_k3,lstm,mixture,bloom_pool,bloom_lstm'); ap.add_argument('--batches', default='256,1024')
ap.add_argument('--rounds', type=int, default=3)
a = ap.parse_args()
dev = torch.device('cuda:0')
S, D, I, K = a.seq, a.dim, a.items, a.steps
Bmax = max(int(x) for x in a.batches.split(','))
torch.manual_seed(0)
seqs = torch.randint(1, I, ((K + 3) * Bmax, S), device=dev)
pad = torch.randint(0, S, ((K + 3) * Bmax,), device=dev)
seqs[torch.arange(S, device=dev)[None, :] < pad[:, None] // 4] = 0
negs = sample_items(I, ((K + 3) * Bmax, S), random_state=np.random.RandomState(1), device=dev)


def gpu_label():
    try:
        pl = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = 'unknown'
    return {'gpu': torch.cuda.get_device_name(dev), 'power_limit': pl or 'unknown'}


def net_of(arm):
    from spotlight_b200.layers import BloomEmbedding
    from spotlight_b200.sequence.representations import CNNNet, LSTMNet, MixtureLSTMNet, PoolNet
    if arm.startswith('bloom_'):
        emb = BloomEmbedding(I, D, compression_ratio=a.ratio, num_hash_functions=a.hashes, padding_idx=0)
        return (PoolNet if arm == 'bloom_pool' else LSTMNet)(I, D, item_embedding_layer=emb)
    if arm == 'pool':
        return PoolNet(I, D)
    if arm == 'cnn_k3':
        return CNNNet(I, D, kernel_width=3)
    if arm == 'lstm':
        return LSTMNet(I, D)
    return MixtureLSTMNet(I, D, num_mixtures=4)


def models(arm, batch):
    """Two models with one initial state: fused_adam and torch.optim.Adam."""
    from spotlight_b200 import optim
    from spotlight_b200.interactions import SequenceInteractions
    from spotlight_b200.sequence.implicit import ImplicitSequenceModel
    inter = SequenceInteractions(np.zeros((1, S), np.int32), num_items=I)
    ms = []
    for opt in (optim.fused_adam(lr=1e-3), lambda p: torch.optim.Adam(p, lr=1e-3)):
        torch.manual_seed(1)
        m = ImplicitSequenceModel(loss='pointwise', representation=net_of(arm), embedding_dim=D, batch_size=batch,
                                  optimizer_func=opt, use_cuda=True, random_state=np.random.RandomState(0))
        m._initialize(inter)
        ms.append(m)
    ms[1]._net.load_state_dict(ms[0]._net.state_dict())
    routes = [m._route() for m in ms]
    assert routes == (['fused_hashed', 'generic'] if arm.startswith('bloom_') else ['fused', 'fused']), routes
    return dict(zip(('fused_adam', 'torch_adam'), ms))


def step(model, k, batch):
    sl = slice(k * batch, (k + 1) * batch)
    model._optimizer.zero_grad()
    if model._route() == 'generic':
        loss = model._generic_step(seqs[sl], negs[sl], 1)
        loss.backward()
    else:
        loss = model._fused_step(seqs[sl], negs[sl], 1)
    model._optimizer.step()
    return loss


out = {}
for arm in a.arms.split(','):
    for batch in (int(x) for x in a.batches.split(',')):
        ms = models(arm, batch)
        res = {name: {'first_losses': [float(step(m, k, batch).detach()) for k in range(2)]} for name, m in ms.items()}
        l0, l1 = res['fused_adam']['first_losses'], res['torch_adam']['first_losses']
        res['first_losses_max_rel_diff'] = max(abs(x - y) / abs(y) for x, y in zip(l0, l1))
        # the same forward on one state, then one update: beyond fp32 rounding the arms compute different things
        assert res['first_losses_max_rel_diff'] <= 1e-5, '%s B=%d: the arms disagree before timing: %s / %s' % (
            arm, batch, l0, l1)
        for m in ms.values():                      # warm-up
            step(m, 2, batch)
        torch.cuda.synchronize()
        times = {r: [] for r in ms}
        for rnd in range(a.rounds):                # alternate the arms
            for name, m in ms.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for k in range(3, 3 + K):
                    r = step(m, k, batch)
                e1.record(); torch.cuda.synchronize()
                times[name].append(e0.elapsed_time(e1) / K)
                res[name]['last_loss'] = float(r.detach())
        for name in ms:
            t = sorted(times[name])[len(times[name]) // 2]
            res[name].update(route=ms[name]._route(), ms_per_step=t, ms_per_step_rounds=times[name],
                             positions_per_s=batch * S / (t * 1e-3))
        res['speedup'] = res['torch_adam']['ms_per_step'] / res['fused_adam']['ms_per_step']
        out['%s_B%d' % (arm, batch)] = res
        print(json.dumps({'%s_B%d' % (arm, batch): res}), flush=True)
        del ms
        torch.cuda.empty_cache()
print(json.dumps({'config': 'adam seq S=%d D=%d items=%d (bloom: ratio=%g H=%d) pointwise' % (S, D, I, a.ratio, a.hashes),
                  **gpu_label(), **out}))
