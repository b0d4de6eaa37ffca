"""Secondary measurement (not bench.py's headline metric): sequence models on a hashed (Bloom) item
table -- the shape of the reference's examples/bloom_embeddings runs scaled to BASELINE.json
configs[4]: 1M items, compression ratio 0.2, 4 hashes, dim 128, S = 200, pointwise loss.

For each representation of --arms (pool, cnn_k3, lstm, mixture with 4 tastes) and each batch of
--batches it times ImplicitSequenceModel's step on two routes from one initial state and the same
minibatches: fused_hashed (one seq_train_step with the row-wise Adagrad applied to the compressed
table and the biases inside, then the optimizer's step for the net's own parameters) against
generic (nn.LSTM / nn.Conv2d / cumsum under autograd over the Bloom gather, the package's loss op,
a dense table gradient and torch.optim.Adagrad).  The routes alternate --rounds times; each
round times --steps steps with CUDA events after two warm-up steps.  Prints ms/step (median
round), positions/s, both routes' first-step loss on the same minibatch, and the GPU's name and
power limit read in the same run.  --items 50000000 --ratio 0.02 gives the configs[3] table size."""
import argparse, json, os, subprocess, sys
import numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from spotlight_b200.sampling import sample_items

ap = argparse.ArgumentParser()
ap.add_argument('--items', type=int, default=1_000_000); ap.add_argument('--ratio', type=float, default=0.2)
ap.add_argument('--hashes', type=int, default=4); ap.add_argument('--dim', type=int, default=128)
ap.add_argument('--seq', type=int, default=200); ap.add_argument('--steps', type=int, default=10)
ap.add_argument('--arms', default='pool,cnn_k3,lstm,mixture'); ap.add_argument('--batches', default='256,1024')
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
    emb = BloomEmbedding(I, D, compression_ratio=a.ratio, num_hash_functions=a.hashes, padding_idx=0)
    if arm == 'pool':
        return PoolNet(I, D, item_embedding_layer=emb)
    if arm == 'cnn_k3':
        return CNNNet(I, D, kernel_width=3, item_embedding_layer=emb)
    if arm == 'lstm':
        return LSTMNet(I, D, item_embedding_layer=emb)
    return MixtureLSTMNet(I, D, num_mixtures=4, item_embedding_layer=emb)


def models(arm, batch):
    """Two models with one initial state: fused_hashed (fused_adagrad) and generic (torch.optim.Adagrad)."""
    from spotlight_b200 import optim
    from spotlight_b200.interactions import SequenceInteractions
    from spotlight_b200.sequence.implicit import ImplicitSequenceModel
    inter = SequenceInteractions(np.zeros((1, S), np.int32), num_items=I)
    ms = []
    for opt in (optim.fused_adagrad(lr=0.05), lambda p: torch.optim.Adagrad(p, lr=0.05)):
        torch.manual_seed(1)
        m = ImplicitSequenceModel(loss='pointwise', representation=net_of(arm), embedding_dim=D, batch_size=batch,
                                  optimizer_func=opt, use_cuda=True, random_state=np.random.RandomState(0))
        m._initialize(inter)
        ms.append(m)
    ms[1]._net.load_state_dict(ms[0]._net.state_dict())
    assert ms[0]._route() == 'fused_hashed' and ms[1]._route() == 'generic'
    return dict(zip(('fused_hashed', 'generic'), ms))


def step(model, route, k, batch):
    sl = slice(k * batch, (k + 1) * batch)
    model._optimizer.zero_grad()
    if route == 'fused_hashed':
        loss = model._fused_step(seqs[sl], negs[sl], 1)
    else:
        loss = model._generic_step(seqs[sl], negs[sl], 1)
        loss.backward()
    model._optimizer.step()
    return loss


out = {}
for arm in a.arms.split(','):
    for batch in (int(x) for x in a.batches.split(',')):
        ms = models(arm, batch)
        res = {}
        for route, m in ms.items():                # first step: same state, same minibatch
            res[route] = {'first_step_loss': float(step(m, route, 0, batch).detach())}
        for route, m in ms.items():                # warm-up
            for k in range(1, 3):
                step(m, route, k, batch)
        torch.cuda.synchronize()
        times = {r: [] for r in ms}
        for rnd in range(a.rounds):                # alternate the routes
            for route, m in ms.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for k in range(3, 3 + K):
                    r = step(m, route, k, batch)
                e1.record(); torch.cuda.synchronize()
                times[route].append(e0.elapsed_time(e1) / K)
                res[route]['last_loss'] = float(r.detach())
        for route in ms:
            t = sorted(times[route])[len(times[route]) // 2]
            res[route].update(ms_per_step=t, ms_per_step_rounds=times[route], positions_per_s=batch * S / (t * 1e-3))
        res['speedup'] = res['generic']['ms_per_step'] / res['fused_hashed']['ms_per_step']
        out['%s_B%d' % (arm, batch)] = res
        del ms
        torch.cuda.empty_cache()
print(json.dumps({'config': 'bloom seq S=%d D=%d items=%d ratio=%g H=%d pointwise' % (S, D, I, a.ratio, a.hashes),
                  **gpu_label(), **out}))
