"""Secondary measurement (not bench.py's headline metric): sequence-model training
step, BASELINE.json configs[4] shape -- 1M items, dim 128, S = 200, pointwise loss,
PoolNet and CNNNet(k=3, 1 layer).  Prints positions/s (CUDA events, K steps).

The lstm arm times ImplicitSequenceModel's LSTMNet step at the same shape for each batch of
--lstm-batches: the fused route (one seq_train_step with the row-wise Adagrad inside, then the
optimizer's step for the LSTM parameters) against the generic route (nn.LSTM under autograd,
the package's loss op, torch.optim.Adagrad), both from the same initial state, alternating
--rounds times.  It prints each route's first-step loss on the same minibatch, and the GPU's
name and power limit.  --profile DIR instead records the fused LSTM step's per-kernel CUDA
times with torch.profiler (a separate run: tracing slows the host)."""
import argparse, json, os, subprocess, sys
import numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from spotlight_b200 import ops
from spotlight_b200.sampling import sample_items

ap = argparse.ArgumentParser()
ap.add_argument('--batch', type=int, default=1024); ap.add_argument('--steps', type=int, default=20)
ap.add_argument('--items', type=int, default=1_000_000); ap.add_argument('--dim', type=int, default=128)
ap.add_argument('--seq', type=int, default=200)
ap.add_argument('--arms', default='pool,cnn_k3,lstm'); ap.add_argument('--lstm-batches', default='256,1024')
ap.add_argument('--rounds', type=int, default=3); ap.add_argument('--profile', default=None)
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
for name, spec in ((n, sp) for n, sp in (('pool', None),
                   ('cnn_k3', dict(kernel_width=[3], dilation=[1], nonlinearity='tanh', residual=True,
                                   weights=[torch.randn(D, D, 3, 1, device=dev) * 0.05],
                                   biases=[torch.zeros(D, device=dev)]))) if n in a.arms.split(',')):
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


def gpu_label():
    try:
        pl = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = 'unknown'
    return {'gpu': torch.cuda.get_device_name(dev), 'power_limit': pl or 'unknown'}


def lstm_models(batch):
    """Two LSTMNet models with one initial state: fused route (fused_adagrad) and generic route
    (torch.optim.Adagrad)."""
    from spotlight_b200 import optim
    from spotlight_b200.interactions import SequenceInteractions
    from spotlight_b200.sequence.implicit import ImplicitSequenceModel
    inter = SequenceInteractions(np.zeros((1, S), np.int32), num_items=I)
    ms = []
    for opt in (optim.fused_adagrad(lr=0.05), lambda p: torch.optim.Adagrad(p, lr=0.05)):
        m = ImplicitSequenceModel(loss='pointwise', representation='lstm', embedding_dim=D, batch_size=batch,
                                  optimizer_func=opt, use_cuda=True, random_state=np.random.RandomState(0))
        m._initialize(inter)
        ms.append(m)
    ms[1]._net.load_state_dict(ms[0]._net.state_dict())
    assert ms[0]._route() == 'fused'
    return ms


def lstm_step(model, route, k, batch):
    sl = slice(k * batch, (k + 1) * batch)
    model._optimizer.zero_grad()
    if route == 'fused':
        loss = model._fused_step(seqs[sl], negs[sl], 1)
    else:
        loss = model._generic_step(seqs[sl], negs[sl], 1)
        loss.backward()
    model._optimizer.step()
    return loss


if a.profile:
    from torch.profiler import ProfilerActivity, profile
    batch = int(a.lstm_batches.split(',')[0])
    fused_m, _ = lstm_models(batch)
    for k in range(3):
        lstm_step(fused_m, 'fused', k, batch)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for k in range(3, 3 + K):
            lstm_step(fused_m, 'fused', k, batch)
        torch.cuda.synchronize()
    os.makedirs(a.profile, exist_ok=True)
    rows = [(e.key, e.device_time_total / K / 1e3, e.count // K) for e in prof.key_averages() if e.device_time_total > 0]
    rows.sort(key=lambda r: -r[1])
    table = {'config': 'lstm fused step S=%d D=%d items=%d B=%d pointwise, %d steps' % (S, D, I, batch, K),
             **gpu_label(), 'ms_per_step_by_kernel': {k: [round(ms, 4), n] for k, ms, n in rows}}
    with open(os.path.join(a.profile, 'lstm_kernels_B%d.json' % batch), 'w') as f:
        json.dump(table, f, indent=1)
    print(json.dumps(table))
    sys.exit(0)

if 'lstm' in a.arms.split(','):
    for batch in (int(x) for x in a.lstm_batches.split(',')):
        assert (K + 3) * batch <= seqs.shape[0]
        models = dict(zip(('fused', 'generic'), lstm_models(batch)))
        res = {}
        for route, m in models.items():            # first step: same state, same minibatch
            res[route] = {'first_step_loss': float(lstm_step(m, route, 0, batch).detach())}
        for route, m in models.items():            # warm-up
            for k in range(1, 3):
                lstm_step(m, route, k, batch)
        torch.cuda.synchronize()
        times = {r: [] for r in models}
        for rnd in range(a.rounds):                # alternate the routes
            for route, m in models.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for k in range(3, 3 + K):
                    r = lstm_step(m, route, k, batch)
                e1.record(); torch.cuda.synchronize()
                times[route].append(e0.elapsed_time(e1) / K)
                res[route]['last_loss'] = float(r.detach())
        for route in models:
            ms = sorted(times[route])[len(times[route]) // 2]
            res[route].update(ms_per_step=ms, ms_per_step_rounds=times[route], positions_per_s=batch * S / (ms * 1e-3))
        out['lstm_B%d' % batch] = res
        del models
        torch.cuda.empty_cache()
print(json.dumps({'config': 'seq S=%d D=%d items=%d B=%d pointwise' % (S, D, I, B), **gpu_label(), **out}))
