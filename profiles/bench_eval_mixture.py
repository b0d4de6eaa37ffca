"""Secondary measurement (not bench.py's headline metric): MixtureLSTMNet evaluation scoring.

Shape: 1M items, D = 128, M = 4, S = 200, 4096 sequences, blocks of 256 (the scorers' default);
``--bloom`` puts a BloomEmbedding item layer under the net.  On one block of sequences, with
CUDA events (median over ``--reps`` runs after warm-up, the arms alternated in one process):

* ``kernel``    slb_mixture_scores alone, item matrix and representation prepared;
* ``two_pass``  an FP32 cuBLAS GEMM (TF32 off) of the (R*2M, D) representation rows against an
                item chunk, then the softmax / combine in torch ops, chunk by chunk;
* ``generic``   _generic_block, the route the scorers took before: the net's own forward() over
                item chunks of 2^18 pairs.

Before timing, the three arms' score blocks must agree (rtol 1e-5 plus 1e-5 of the row's largest
|score|) and so must their slb_rank_targets average ranks, up to the items whose scores lie within
that tolerance of the target's.  Then sequence_mrr_score over all sequences end to end.  Reports
the kernel's FLOP/s (2 * R * I * 2M * D over kernel time) against the H100 SXM data-sheet FP32
rate, and the card's name and power limit read in the same run.  Prints one JSON line."""
import argparse, json, os, subprocess, sys, time
import numpy as np, torch
import torch.nn.functional as F
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from spotlight_b200 import _lib, evaluation as ev, ops
from spotlight_b200.interactions import SequenceInteractions
from spotlight_b200.layers import BloomEmbedding
from spotlight_b200.sequence.implicit import ImplicitSequenceModel
from spotlight_b200.sequence.representations import MixtureLSTMNet

FP32_DATASHEET = 67e12           # FLOP/s, H100 SXM data sheet, dense FP32 (non-tensor)

ap = argparse.ArgumentParser()
ap.add_argument('--items', type=int, default=1_000_000); ap.add_argument('--dim', type=int, default=128)
ap.add_argument('--mixtures', type=int, default=4); ap.add_argument('--seq-len', type=int, default=200)
ap.add_argument('--seqs', type=int, default=4096); ap.add_argument('--block', type=int, default=256)
ap.add_argument('--reps', type=int, default=20); ap.add_argument('--chunk', type=int, default=1 << 16)
ap.add_argument('--bloom', action='store_true')
a = ap.parse_args()
assert torch.cuda.is_available(), 'bench_eval_mixture.py measures on a CUDA device'
torch.backends.cuda.matmul.allow_tf32 = False
torch.set_grad_enabled(False)    # evaluation: no arm may record an autograd graph
dev = torch.device('cuda:0')
I, D, M, R = a.items, a.dim, a.mixtures, a.block
rs = np.random.RandomState(0)
seqs = rs.randint(1, I, (a.seqs, a.seq_len + 1)).astype(np.int32)
inter = SequenceInteractions(seqs, num_items=I)
torch.manual_seed(0)
emb = BloomEmbedding(I, D, padding_idx=0) if a.bloom else None
model = ImplicitSequenceModel(representation=MixtureLSTMNet(I, D, num_mixtures=M, item_embedding_layer=emb),
                              embedding_dim=D, use_cuda=True, random_state=np.random.RandomState(1))
model._initialize(inter)
net = model._net
net.projection.weight.mul_(8.0)  # mixture weights away from uniform, as a trained model's
net.item_biases.weight.normal_(0, 0.1)
net.train(False)
out = {'config': 'mixture eval items=%d dim=%d M=%d S=%d sequences=%d block=%d%s'
                 % (I, D, M, a.seq_len, a.seqs, R, ' bloom' if a.bloom else '')}

lib = _lib.load()
blk = torch.from_numpy(seqs[:R, :-1].astype(np.int64)).to(dev)
targets = torch.from_numpy(seqs[:R, -1].astype(np.int64)).to(dev)
final = net.user_representation(blk)[1]
reps = final.reshape(R, 2 * M, D).contiguous()
items = ev._item_matrix(net.item_embeddings, I, dev).contiguous()
bias = net.item_biases.weight.reshape(-1).contiguous()
st = ops._stream()
kout = torch.empty(R, I, device=dev)
tout = torch.empty(R, I, device=dev)


def kernel():
    _lib.check(lib.slb_mixture_scores(ops._ptr(reps), R, M, D, ops._ptr(items), ops._ptr(bias), I,
                                      ops._ptr(kout), st), 'mixture_scores')
    return kout


def two_pass():
    A = reps.reshape(R * 2 * M, D)
    for lo in range(0, I, a.chunk):
        hi = min(I, lo + a.chunk)
        x = (A @ items[lo:hi].t()).view(R, 2 * M, hi - lo)
        w = F.softmax(x[:, M:], dim=1)
        tout[:, lo:hi] = (w * x[:, :M]).sum(1) + bias[lo:hi]
    return tout


def generic():
    return ev._generic_block(lambda r, t: net(r, t.reshape(-1, 1)), final, I, dev)


arms = {'kernel': kernel, 'two_pass': two_pass, 'generic': generic}

# ---- agreement of the score blocks and of their rankings
blocks = {k: fn().clone() for k, fn in arms.items()}
ref = blocks['kernel'].double()
rowmax = ref.abs().amax(1, keepdim=True)
tol = 1e-5 * ref.abs() + 1e-5 * rowmax
row_ptr = np.arange(R + 1)
ranks = {k: ev._rank_targets(b, row_ptr, targets.cpu().numpy(), avg_rank=True)[0] for k, b in blocks.items()}
s_t = ref.gather(1, targets.view(-1, 1))
ambiguous = ((ref - s_t).abs() <= 1e-5 * s_t.abs() + 1e-5 * rowmax).sum(1).cpu().numpy()   # target included
agree = {}
for k in ('two_pass', 'generic'):
    err = (blocks[k].double() - ref).abs()
    d_rank = np.abs(ranks[k] - ranks['kernel'])
    agree[k] = {'max_abs_err': float(err.max()), 'within_tol': bool((err <= tol).all()),
                'max_rank_diff': float(d_rank.max()), 'ranks_equal': int((d_rank == 0).sum()),
                'ranks_within_ambiguity': bool((d_rank <= ambiguous - 1).all())}
    assert agree[k]['within_tol'] and agree[k]['ranks_within_ambiguity'], (k, agree[k])
out['agreement_vs_kernel'] = agree
del blocks, ref, tol
torch.cuda.empty_cache()

# ---- one block, CUDA events, arms alternated
ms = {k: [] for k in arms}
for rep in range(a.reps + 1):
    for k, fn in arms.items():
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record(); torch.cuda.synchronize()
        if rep >= 1:
            ms[k].append(e0.elapsed_time(e1))
flop = 2.0 * R * I * 2 * M * D
for k in arms:
    out[k] = {'ms_median': float(np.median(ms[k])), 'ms_min': float(np.min(ms[k])), 'runs': len(ms[k])}
kt = out['kernel']['ms_median'] * 1e-3
out['kernel'].update({'flop': flop, 'tflop_per_s': flop / kt / 1e12,
                      'share_of_datasheet_fp32': flop / kt / FP32_DATASHEET, 'bound': 'compute (FP32 FMA)'})
out['speedup_vs_two_pass'] = out['two_pass']['ms_median'] / out['kernel']['ms_median']
out['speedup_vs_generic'] = out['generic']['ms_median'] / out['kernel']['ms_median']


# ---- end to end: sequence_mrr_score over every sequence on the new path
def sync_time(fn):
    torch.cuda.synchronize(); t = time.perf_counter(); r = fn(); torch.cuda.synchronize()
    return time.perf_counter() - t, r


ev.sequence_mrr_score(model, SequenceInteractions(seqs[:R], num_items=I), sequence_block=R)
t_e2e, mrr = sync_time(lambda: ev.sequence_mrr_score(model, inter, sequence_block=R))
out['sequence_mrr_score'] = {'s': t_e2e, 'sequences_per_s': a.seqs / t_e2e, 'mean': float(mrr.mean())}

try:
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                       capture_output=True, text=True, timeout=30).stdout.strip().split('\n')[0]
except (OSError, subprocess.SubprocessError):
    q = 'unknown'
out['card'] = {'torch_name': torch.cuda.get_device_name(0), 'nvidia_smi_name_power_limit': q}
print(json.dumps(out))
