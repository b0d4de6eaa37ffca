"""Secondary measurement (not bench.py's headline metric): evaluation on the device.

BASELINE.json configs[1] shape (1M users x 100K items x dim 64, a synthetic test set with train
exclusions): mrr_score and precision_recall_score(k=[1, 10, 100]) end to end in users/s; on
one user block, the block GEMM, slb_rank_targets and slb_rank_pairs alone (CUDA events, the two
ranking kernels alternated in the same run), with slb_rank_targets' algorithmic bytes over the
H100 SXM data-sheet HBM3 bandwidth.  configs[4] shape (1M items x dim 128, S = 200):
sequence_mrr_score over a block of sequences.  The reference's per-user loop (predict +
rankdata) is timed on a few users and extrapolated.  Prints one JSON line with the card's name
and power limit."""
import argparse, json, os, subprocess, sys, time
import numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from spotlight_b200 import _lib, evaluation as ev, ops
from spotlight_b200.factorization.implicit import ImplicitFactorizationModel
from spotlight_b200.interactions import Interactions, SequenceInteractions
from spotlight_b200.sequence.implicit import ImplicitSequenceModel

HBM_DATASHEET = 3.35e12          # bytes/s, H100 SXM data sheet

ap = argparse.ArgumentParser()
ap.add_argument('--users', type=int, default=1_000_000); ap.add_argument('--items', type=int, default=100_000)
ap.add_argument('--dim', type=int, default=64); ap.add_argument('--test-per-user', type=int, default=5)
ap.add_argument('--train-per-user', type=int, default=20); ap.add_argument('--user-block', type=int, default=2048)
ap.add_argument('--kernel-reps', type=int, default=20); ap.add_argument('--ref-users', type=int, default=50)
ap.add_argument('--seq-items', type=int, default=1_000_000); ap.add_argument('--seq-dim', type=int, default=128)
ap.add_argument('--seq-len', type=int, default=200); ap.add_argument('--seqs', type=int, default=4096)
ap.add_argument('--seq-block', type=int, default=256)
a = ap.parse_args()
assert torch.cuda.is_available(), 'bench_eval.py measures on a CUDA device'
dev = torch.device('cuda:0')
U, I, D = a.users, a.items, a.dim
rs = np.random.RandomState(0)


def sync_time(fn):
    torch.cuda.synchronize(); t = time.perf_counter(); r = fn(); torch.cuda.synchronize()
    return time.perf_counter() - t, r


def interactions(per_user):
    return Interactions(np.repeat(np.arange(U, dtype=np.int32), per_user), rs.randint(0, I, U * per_user).astype(np.int32),
                        num_users=U, num_items=I)


train, test = interactions(a.train_per_user), interactions(a.test_per_user)
model = ImplicitFactorizationModel(loss='bpr', embedding_dim=D, use_cuda=True, random_state=np.random.RandomState(1))
model._initialize(train)
out = {'config': 'eval users=%d items=%d dim=%d test/user=%d train/user=%d block=%d'
                 % (U, I, D, a.test_per_user, a.train_per_user, a.user_block)}

# ---- end to end (warm-up on a small slice first: module load, cuBLAS algorithm choice)
small = Interactions(test.user_ids[:a.user_block * a.test_per_user], test.item_ids[:a.user_block * a.test_per_user],
                     num_users=U, num_items=I)
ev.mrr_score(model, small, train); ev.precision_recall_score(model, small, train, k=[1, 10, 100])
t_mrr, mrr = sync_time(lambda: ev.mrr_score(model, test, train, user_block=a.user_block))
t_pr, (p, r) = sync_time(lambda: ev.precision_recall_score(model, test, train, k=[1, 10, 100], user_block=a.user_block))
out['mrr_score'] = {'s': t_mrr, 'users_per_s': U / t_mrr, 'mean': float(mrr.mean())}
out['precision_recall_score_k1_10_100'] = {'s': t_pr, 'users_per_s': U / t_pr,
                                           'mean_precision': p.mean(0).tolist(), 'mean_recall': r.mean(0).tolist()}

# ---- one block: GEMM, slb_rank_targets, slb_rank_pairs (alternated), CUDA events
lib = _lib.load()
blk = np.arange(a.user_block, dtype=np.int64)
users_d = torch.from_numpy(blk).to(dev)
tr, te = train.tocsr()[blk], test.tocsr()[blk]
scores = ev._score_block(model, users_d)
ev._exclude(scores, np.repeat(np.arange(len(blk)), np.diff(tr.indptr)), tr.indices)
rp = torch.from_numpy(te.indptr.astype(np.int64)).to(dev)
tg = torch.from_numpy(te.indices.astype(np.int64)).to(dev)
prow = torch.from_numpy(np.repeat(np.arange(len(blk)), np.diff(te.indptr)).astype(np.int64)).to(dev)
n_t = tg.numel()
avg = torch.empty(n_t, device=dev); pos = torch.empty(n_t, dtype=torch.int64, device=dev)
ranks = torch.empty(n_t, device=dev)
st = ops._stream()
runs = {
    'gemm_block': lambda: ev._score_block(model, users_d),
    'rank_targets': lambda: lib.slb_rank_targets(ops._ptr(scores), len(blk), I, ops._ptr(rp), ops._ptr(tg), n_t,
                                                 ops._ptr(avg), ops._ptr(pos), st),
    'rank_pairs': lambda: lib.slb_rank_pairs(ops._ptr(scores), len(blk), I, ops._ptr(prow), ops._ptr(tg), n_t,
                                             ops._ptr(ranks), st),
}
ms = {k: [] for k in runs}
for rep in range(a.kernel_reps + 2):
    for k, fn in runs.items():
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record(); torch.cuda.synchronize()
        if rep >= 2:
            ms[k].append(e0.elapsed_time(e1))
assert torch.equal(avg, ranks), 'rank_targets and rank_pairs disagree'
bytes_rt = 4 * I * len(blk) + n_t * (8 + 4 + 4 + 8) + 8 * (len(blk) + 1)   # row once per chunk (1 chunk) + targets
for k in runs:
    out[k] = {'ms_median': float(np.median(ms[k])), 'ms_min': float(np.min(ms[k]))}
out['rank_targets']['algorithmic_bytes'] = bytes_rt
out['rank_targets']['share_of_datasheet_hbm'] = bytes_rt / (out['rank_targets']['ms_median'] * 1e-3) / HBM_DATASHEET
out['rank_pairs']['algorithmic_bytes'] = 4 * I * n_t

# ---- the reference's loop (predict + rankdata per user), a few users, extrapolated
import scipy.stats as sst
tcsr, trcsr = test.tocsr(), train.tocsr()


def ref_loop():
    for u in range(a.ref_users):
        pr = -model.predict(u)
        pr[trcsr[u].indices] = ev.FLOAT_MAX
        (1.0 / sst.rankdata(pr)[tcsr[u].indices]).mean()


ref_loop()
t_ref, _ = sync_time(ref_loop)
out['reference_loop_mrr'] = {'users_timed': a.ref_users, 's_per_user': t_ref / a.ref_users,
                             'extrapolated_s_all_users': t_ref / a.ref_users * U}
del scores, model, train, test, tr, te, tcsr, trcsr
torch.cuda.empty_cache()

# ---- configs[4] shape: sequence_mrr_score over a block of sequences
SI, S = a.seq_items, a.seq_len
seqs = rs.randint(1, SI, (a.seqs, S + 1)).astype(np.int32)
sinter = SequenceInteractions(seqs, num_items=SI)
smodel = ImplicitSequenceModel(representation='pooling', embedding_dim=a.seq_dim, use_cuda=True,
                               random_state=np.random.RandomState(2))
smodel._initialize(sinter)
warm = SequenceInteractions(seqs[:a.seq_block], num_items=SI)
ev.sequence_mrr_score(smodel, warm, sequence_block=a.seq_block)
t_seq, smrr = sync_time(lambda: ev.sequence_mrr_score(smodel, sinter, sequence_block=a.seq_block))
out['sequence_mrr_score'] = {'config': 'pooling items=%d dim=%d S=%d sequences=%d block=%d'
                                       % (SI, a.seq_dim, S, a.seqs, a.seq_block),
                             's': t_seq, 'sequences_per_s': a.seqs / t_seq, 'mean': float(smrr.mean())}

try:
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                       capture_output=True, text=True, timeout=30).stdout.strip().split('\n')[0]
except (OSError, subprocess.SubprocessError):
    q = 'unknown'
out['card'] = {'torch_name': torch.cuda.get_device_name(0), 'nvidia_smi_name_power_limit': q}
print(json.dumps(out))
