"""Secondary measurement (not bench.py's headline metric): ImplicitSequenceModel's MixtureLSTMNet
training step at BASELINE.json configs[4]'s shape -- 1M items, dim 128, S = 200, M = 4 mixtures,
pointwise loss, row-wise Adagrad.

For each batch of --batches it times the fused route (one seq_train_step with the Adagrad update of
the item table inside, then the optimizer's step for the LSTM and projection parameters) against the
generic route (nn.LSTM, nn.Conv1d and the softmax head under autograd, the package's loss op,
torch.optim.Adagrad), both from the same initial state, alternating --rounds times, and reports
each route's median ms per step (CUDA events over --steps steps), its first-step loss on the same
minibatch and the GPU's name and power limit.  --profile DIR instead records one fused step's CUDA
time by kernel with torch.profiler and splits it into the recurrence, the k = 1 GEMMs (the LSTM's
four gate blocks and the 2M projection blocks, forward and backward), the
mixture head, the item-table reduction and the rest (a separate run: tracing slows the host)."""
import argparse, json, os, subprocess, sys
import numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from spotlight_b200.sampling import sample_items

ap = argparse.ArgumentParser()
ap.add_argument('--batches', default='256,1024'); ap.add_argument('--steps', type=int, default=10)
ap.add_argument('--items', type=int, default=1_000_000); ap.add_argument('--dim', type=int, default=128)
ap.add_argument('--seq', type=int, default=200); ap.add_argument('--mixtures', type=int, default=4)
ap.add_argument('--rounds', type=int, default=3); ap.add_argument('--profile', default=None)
a = ap.parse_args()
dev = torch.device('cuda:0')
S, D, I, K, M = a.seq, a.dim, a.items, a.steps, a.mixtures
batches = [int(x) for x in a.batches.split(',')]
torch.manual_seed(0)
nseq = (K + 3) * max(batches)
seqs = torch.randint(1, I, (nseq, S), device=dev)
pad = torch.randint(0, S, (nseq,), device=dev)
seqs[torch.arange(S, device=dev)[None, :] < pad[:, None] // 4] = 0
negs = sample_items(I, (nseq, S), random_state=np.random.RandomState(1), device=dev)


def gpu_label():
    try:
        pl = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = 'unknown'
    return {'gpu': torch.cuda.get_device_name(dev), 'power_limit': pl or 'unknown'}


def models(batch, routes=('fused', 'generic')):
    """MixtureLSTMNet models with one initial state: fused route (fused_adagrad) and generic route
    (torch.optim.Adagrad)."""
    from spotlight_b200 import optim
    from spotlight_b200.interactions import SequenceInteractions
    from spotlight_b200.sequence.implicit import ImplicitSequenceModel
    from spotlight_b200.sequence.representations import MixtureLSTMNet
    inter = SequenceInteractions(np.zeros((1, S), np.int32), num_items=I)
    opts = dict(fused=optim.fused_adagrad(lr=0.05), generic=lambda p: torch.optim.Adagrad(p, lr=0.05))
    out = {}
    for r in routes:
        torch.manual_seed(0)
        m = ImplicitSequenceModel(loss='pointwise', representation=MixtureLSTMNet(I, D, num_mixtures=M),
                                  embedding_dim=D, batch_size=batch, optimizer_func=opts[r], use_cuda=True,
                                  random_state=np.random.RandomState(0))
        m._initialize(inter)
        out[r] = m
    assert out.get('fused') is None or out['fused']._route() == 'fused'
    return out


def step(model, route, k, batch):
    sl = slice(k * batch, (k + 1) * batch)
    model._optimizer.zero_grad()
    if route == 'fused':
        loss = model._fused_step(seqs[sl], negs[sl], 1)
    else:
        loss = model._generic_step(seqs[sl], negs[sl], 1)
        loss.backward()
    model._optimizer.step()
    return loss


# kernel-name fragments of each part of the fused step
PARTS = [('recurrence', ('lstm_fwd', 'lstm_bwd')),
         ('k1_gemms', ('conv_gemm', 'conv_dw', 'conv_wt', 'seq_gather')),   # LSTM gate blocks and projection
         ('mixture_head', ('mix_score',)),
         ('item_reduce', ('seg_', 'seq_fill', 'seq_reduce'))]

if a.profile:
    from torch.profiler import ProfilerActivity, profile
    batch = batches[0]
    m = models(batch, ('fused',))['fused']
    for k in range(3):
        step(m, 'fused', k, batch)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for k in range(3, 3 + K):
            step(m, 'fused', k, batch)
        torch.cuda.synchronize()
    rows = [(e.key, e.device_time_total / K / 1e3, e.count // K) for e in prof.key_averages() if e.device_time_total > 0]
    rows.sort(key=lambda r: -r[1])
    split = {p: 0.0 for p, _ in PARTS}
    split['other'] = 0.0
    for key, ms, _ in rows:
        part = next((p for p, frags in PARTS if any(f in key for f in frags)), 'other')
        split[part] += ms
    table = {'config': 'mixture fused step S=%d D=%d M=%d items=%d B=%d pointwise adagrad, %d steps'
                       % (S, D, M, I, batch, K),
             **gpu_label(), 'ms_per_step_by_part': {p: round(v, 4) for p, v in split.items()},
             'ms_per_step_by_kernel': {k: [round(ms, 4), n] for k, ms, n in rows}}
    os.makedirs(a.profile, exist_ok=True)
    with open(os.path.join(a.profile, 'mixture_kernels_B%d.json' % batch), 'w') as f:
        json.dump(table, f, indent=1)
    print(json.dumps({k: v for k, v in table.items() if k != 'ms_per_step_by_kernel'}))
    sys.exit(0)

out = {}
for batch in batches:
    ms_ = models(batch)
    res = {}
    for route, m in ms_.items():                 # first step: same state, same minibatch
        res[route] = {'first_step_loss': float(step(m, route, 0, batch).detach())}
    for route, m in ms_.items():                 # warm-up
        for k in range(1, 3):
            step(m, route, k, batch)
    torch.cuda.synchronize()
    times = {r: [] for r in ms_}
    for rnd in range(a.rounds):                  # alternate the routes
        for route, m in ms_.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for k in range(3, 3 + K):
                r = step(m, route, k, batch)
            e1.record(); torch.cuda.synchronize()
            times[route].append(e0.elapsed_time(e1) / K)
            res[route]['last_loss'] = float(r.detach())
    for route in ms_:
        med = sorted(times[route])[len(times[route]) // 2]
        res[route].update(ms_per_step=med, ms_per_step_rounds=times[route], positions_per_s=batch * S / (med * 1e-3))
    res['speedup'] = res['generic']['ms_per_step'] / res['fused']['ms_per_step']
    out['mixture_B%d' % batch] = res
    del ms_
    torch.cuda.empty_cache()
print(json.dumps({'config': 'mixture S=%d D=%d M=%d items=%d pointwise adagrad' % (S, D, M, I), **gpu_label(), **out}))
