"""Secondary measurement (not bench.py's headline metric): sequence-model training
step, BASELINE.json configs[4] shape -- 1M items, dim 128, S = 200, pointwise loss,
PoolNet and CNNNet(k=3, 1 layer).  Prints positions/s (CUDA events, K steps)."""
import argparse, json, os, sys
import numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from spotlight_b200 import ops
from spotlight_b200.sampling import sample_items

ap = argparse.ArgumentParser()
ap.add_argument('--batch', type=int, default=1024); ap.add_argument('--steps', type=int, default=20)
ap.add_argument('--items', type=int, default=1_000_000); ap.add_argument('--dim', type=int, default=128)
ap.add_argument('--seq', type=int, default=200)
a = ap.parse_args()
dev = torch.device('cuda:0')
B, S, D, I, K = a.batch, a.seq, a.dim, a.items, a.steps
torch.manual_seed(0)
E = torch.randn(I, D, device=dev) / D; E[0] = 0
bias = torch.zeros(I, 1, device=dev)
seqs = torch.randint(1, I, ((K + 3) * B, S), device=dev)
pad = torch.randint(0, S, ((K + 3) * B,), device=dev)
seqs[torch.arange(S, device=dev)[None, :] < pad[:, None] // 4] = 0
negs = sample_items(I, ((K + 3) * B, S), random_state=np.random.RandomState(1), device=dev)
out = {}
for name, spec in (('pool', None),
                   ('cnn_k3', dict(kernel_width=[3], dilation=[1], nonlinearity='tanh', residual=True,
                                   weights=[torch.randn(D, D, 3, 1, device=dev) * 0.05],
                                   biases=[torch.zeros(D, device=dev)]))):
    from spotlight_b200 import _lib
    sE, sb = torch.zeros_like(E), torch.zeros_like(bias)
    fused = None if os.environ.get('SEQ_DENSE') else dict(kind=_lib.OPT_ADAGRAD, lr=0.05, weight_decay=0.0, eps=1e-10,
                                                       state_E=sE, state_bias=sb)

    def step(k):
        # default: row-wise Adagrad fused into the step (no dense 512 MB item-table gradient);
        # SEQ_DENSE=1: the round-1 measurement (dense dE / dbias, no optimizer)
        sl = slice(k * B, (k + 1) * B)
        return ops.seq_train_step(E, bias, seqs[sl], negs[sl], 'pointwise', 1, spec, fused=fused)
    for k in range(3):
        step(k)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for k in range(3, 3 + K):
        r = step(k)
    e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / K
    out[name] = {'ms_per_step': ms, 'positions_per_s': B * S / (ms * 1e-3), 'loss': float(r['loss'])}
print(json.dumps({'config': 'seq S=%d D=%d items=%d B=%d pointwise' % (S, D, I, B), **out}))
