"""Shared driver for the sharded-step tests (CPU/gloo with a NumPy backend,
GPU/NCCL with the product backend): spawns a process group of `world` ranks, runs a
few global steps on it and on a single-process oracle, and returns both parameter sets."""

import os
import shutil
import tempfile

import numpy as np
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle import mf as omf
from oracle import seq as oseq


def _rank_main(rank, world, store, q, backend, job, args):
    try:
        if backend == 'nccl':
            torch.cuda.set_device(rank)
            dev = torch.device('cuda', rank)
            dist.init_process_group('nccl', init_method=store, rank=rank, world_size=world, device_id=dev)
        else:
            dev = torch.device('cpu')
            dist.init_process_group('gloo', init_method=store, rank=rank, world_size=world)
        out = job(rank, world, dev, *args)
        if backend == 'nccl':
            torch.cuda.synchronize()
        q.put((rank, out, None))
    except Exception:                        # surface the traceback in the parent
        import traceback
        q.put((rank, None, traceback.format_exc()))
    finally:
        if dist.is_initialized():
            dist.destroy_process_group()


def run_world(job, world, args=(), backend='gloo', timeout=300):
    """Runs ``job(rank, world, device, *args)`` (a module-level function) on ``world`` spawned
    ranks of one process group -- ``gloo`` on the CPU, or ``nccl`` with rank r on GPU r.  Returns
    {rank: result}; a rank that raises fails the caller with its traceback.

    The ranks meet through a file in a fresh temporary directory rather than on a TCP port, so
    a port some other socket holds cannot stall or fail the group; ranks still running when the
    call fails are terminated, so none outlives it."""
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    rendezvous = tempfile.mkdtemp(prefix='sharded_world_')
    store = 'file://' + os.path.join(rendezvous, 'store')
    procs = [ctx.Process(target=_rank_main, args=(r, world, store, q, backend, job, tuple(args)))
             for r in range(world)]
    try:
        for p in procs:
            p.start()
        res = {}
        for _ in range(world):
            rank, out, err = q.get(timeout=timeout)
            assert err is None, 'rank %d failed:\n%s' % (rank, err)
            res[rank] = out
        for p in procs:
            p.join(timeout=120)
            assert p.exitcode == 0
        return res
    finally:
        for p in procs:
            if p.is_alive():
                p.terminate()
                p.join()
        shutil.rmtree(rendezvous, ignore_errors=True)


def gather_rows(shard, chunk, n):
    """The first ``n`` rows of a range-sharded table, as NumPy, from every rank's ``shard`` of at
    most ``chunk`` rows: each padded to ``chunk`` rows, all-gathered and concatenated in rank order."""
    pad = shard.new_zeros((chunk,) + tuple(shard.shape[1:]))
    pad[:shard.shape[0]] = shard
    parts = [torch.empty_like(pad) for _ in range(dist.get_world_size())]
    dist.all_gather(parts, pad)
    return torch.cat(parts)[:n].cpu().numpy()


class NumpyBackend(object):
    """Oracle stand-in for spotlight_b200.sharded.GpuBackend (tests only)."""

    def unique_bucket(self, ids, rows, chunk, nparts):
        x = ids.numpy()
        uniq, inverse = np.unique(x, return_inverse=True)
        bounds = [int(np.searchsorted(uniq, p * chunk)) for p in range(nparts)] + [len(uniq)]
        return torch.from_numpy(uniq), torch.from_numpy(inverse.astype(np.int64)), bounds

    def gather(self, W, b, local_ids):
        i = local_ids.numpy()
        return torch.from_numpy(W.numpy()[i].copy()), torch.from_numpy(b.numpy()[i].copy())

    def local_step(self, st, cache_rows, cache_bias, n_cache, users_local, pos_idx, neg_idx, loss,
                   global_batch, n_neg=1):
        B = users_local.numel()
        r = omf.mf_step(st.Wu.numpy().astype(np.float64), cache_rows.numpy().astype(np.float64),
                        st.bu.numpy().astype(np.float64), cache_bias.numpy().astype(np.float64),
                        users_local.numpy(), pos_idx.numpy(), neg_idx.numpy(), loss, n_neg, np.float64)
        scale = B / float(global_batch)
        for W, S, g in ((st.Wu, st.sWu, r['dWu'] * scale), (st.bu, st.sbu, r['dbu'].reshape(-1) * scale)):
            s = S.numpy().astype(np.float64) + g * g
            w = W.numpy().astype(np.float64) - st.lr * g / (np.sqrt(s) + st.eps)
            S.copy_(torch.from_numpy(s.astype(np.float32)))
            W.copy_(torch.from_numpy(w.astype(np.float32)))
        return (torch.tensor(float(r['loss']) * scale, dtype=torch.float32),
                torch.from_numpy((r['dWi'] * scale).astype(np.float32))[:n_cache],
                torch.from_numpy((r['dbi'].reshape(-1) * scale).astype(np.float32))[:n_cache])

    # hashed item table (config 4)
    def bloom_local_step(self, st, W_full, users_local, items, negs, loss, global_batch):
        H = len(st.item_seeds)
        B = users_local.numel()
        r = omf.mf_bloom_step(st.Wu.numpy().astype(np.float64), W_full.numpy().astype(np.float64),
                              st.bu.numpy().astype(np.float64), st.bi.numpy().astype(np.float64),
                              users_local.numpy(), items.numpy(), negs.numpy(), loss, H, 0, np.float64)
        scale = B / float(global_batch)
        # bias gradients as (id, g) pairs, as the product kernel hands them out; for the oracle the
        # per-id totals are enough: one pair per touched id
        def pairs(dense):
            d = dense.reshape(-1) * scale
            ids = np.nonzero(d)[0]
            return torch.from_numpy(ids.astype(np.int64)), torch.from_numpy(d[ids].astype(np.float32))
        f = lambda x: torch.from_numpy((x * scale).astype(np.float32))       # noqa: E731
        return (torch.tensor(float(r['loss']) * scale, dtype=torch.float32), f(r['dWu']), f(r['dWi']),
                pairs(r['dbu']), pairs(r['dbi']))

    def adagrad_dense(self, W, S, G, lr, eps):
        g = G.numpy().astype(np.float64)
        s = S.numpy().astype(np.float64) + g * g
        w = W.numpy().astype(np.float64) - lr * g / (np.sqrt(s) + eps)
        S.copy_(torch.from_numpy(s.astype(np.float32)))
        W.copy_(torch.from_numpy(w.astype(np.float32)))

    def bias_sparse_adagrad(self, ids, g, bias, state, lr, eps):
        tot = np.zeros(bias.numel())
        np.add.at(tot, ids.numpy(), g.numpy().astype(np.float64))
        s = state.numpy().astype(np.float64) + tot * tot
        w = bias.numpy().astype(np.float64) - lr * tot / (np.sqrt(s) + eps)
        state.copy_(torch.from_numpy(s.astype(np.float32)))
        bias.copy_(torch.from_numpy(w.astype(np.float32)))

    # adaptive hinge pieces
    def scores(self, st, cache_rows, cache_bias, u_idx, i_idx):
        Wu, bu = st.Wu.numpy().astype(np.float64), st.bu.numpy().astype(np.float64)
        Wi, bi = cache_rows.numpy().astype(np.float64), cache_bias.numpy().astype(np.float64)
        u, i = u_idx.numpy(), i_idx.numpy()
        return torch.from_numpy(((Wu[u] * Wi[i]).sum(1) + bu[u] + bi[i]).astype(np.float32))

    def adaptive_loss(self, pos, negmat):
        p, ng = pos.numpy().astype(np.float64), negmat.numpy().astype(np.float64)
        k = ng.argmax(axis=0)                       # first index on ties, as torch.max
        hardest = ng[k, np.arange(len(p))]
        act = ((hardest - p + 1.0) >= 0.0).astype(np.float64)    # sub-gradient 1 at the kink (losses.py:115-124)
        loss = np.maximum(hardest - p + 1.0, 0.0).mean()
        gp = -act / float(len(p))
        gn = np.zeros_like(ng)
        gn[k, np.arange(len(p))] = act / float(len(p))
        return (torch.tensor(loss, dtype=torch.float32), torch.from_numpy(gp.astype(np.float32)),
                torch.from_numpy(gn.astype(np.float32)))

    def scores_backward(self, st, cache_rows, g, u_idx, i_idx):
        Wu, Wi = st.Wu.numpy().astype(np.float64), cache_rows.numpy().astype(np.float64)
        u, i, gg = u_idx.numpy(), i_idx.numpy(), g.numpy().astype(np.float64)
        dWu, dWi = np.zeros_like(Wu), np.zeros_like(Wi)
        dbu, dbi = np.zeros(len(Wu)), np.zeros(len(Wi))
        np.add.at(dWu, u, gg[:, None] * Wi[i])
        np.add.at(dWi, i, gg[:, None] * Wu[u])
        np.add.at(dbu, u, gg)
        np.add.at(dbi, i, gg)
        f = lambda x: torch.from_numpy(x.astype(np.float32))      # noqa: E731
        return f(dWu), f(dWi), f(dbu), f(dbi)

    # epoch-level pieces of the sharded fit(), host NumPy (the reference's own calls)
    def to_device(self, ids):
        return torch.from_numpy(np.ascontiguousarray(ids).astype(np.int64))

    def shuffled_order(self, n, random_state):
        order = np.arange(n)
        random_state.shuffle(order)
        return torch.from_numpy(order)

    def permute(self, order, users, items):
        return users[order], items[order]

    def sample(self, num_items, count, random_state):
        return torch.from_numpy(random_state.randint(0, num_items, count, dtype=np.int64))

    def seq_local_step(self, E_cache, bias_cache, n_cache, seqs_idx, negs_idx, loss, cnn, norm_count):
        E = E_cache.numpy().astype(np.float64)
        b = bias_cache.numpy().astype(np.float64).reshape(-1, 1)
        sq, ng = seqs_idx.numpy(), negs_idx.numpy()
        if cnn is None:
            r = oseq.pool_step(E, b, sq, ng, loss, 1, np.float64)
            dconvs = []
        else:
            convs = [(w.numpy().astype(np.float64), c.numpy().astype(np.float64))
                     for w, c in zip(cnn['weights'], cnn['biases'])]
            r = oseq.cnn_step(E, b, convs, sq, ng, cnn['kernel_width'], cnn['dilation'], loss, 1,
                              cnn['nonlinearity'], cnn['residual'], np.float64)
            dconvs = r['dconvs']
        scale = float((sq != 0).sum()) / float(norm_count.item())
        f = lambda x: torch.from_numpy((x * scale).astype(np.float32))      # noqa: E731
        return (torch.tensor(float(r['loss']) * scale, dtype=torch.float32), f(r['dE'])[:n_cache],
                f(r['dbias'].reshape(-1))[:n_cache], [f(w) for w, _ in dconvs], [f(c) for _, c in dconvs])

    def owner_update(self, st, local_ids, g_rows, g_bias):
        rows = st.Wi.shape[0]
        dW = np.zeros((rows, st.Wi.shape[1]))
        db = np.zeros(rows)
        np.add.at(dW, local_ids.numpy(), g_rows.numpy().astype(np.float64))
        np.add.at(db, local_ids.numpy(), g_bias.numpy().astype(np.float64))
        for W, S, g in ((st.Wi, st.sWi, dW), (st.bi, st.sbi, db)):
            s = S.numpy().astype(np.float64) + g * g
            w = W.numpy().astype(np.float64) - st.lr * g / (np.sqrt(s) + st.eps)
            S.copy_(torch.from_numpy(s.astype(np.float32)))
            W.copy_(torch.from_numpy(w.astype(np.float32)))


def make_problem(seed, U, I, D, B, steps, n_neg=1):
    rs = np.random.RandomState(seed)
    Wu = (rs.randn(U, D) * 0.3).astype(np.float32)
    Wi = (rs.randn(I, D) * 0.3).astype(np.float32)
    bu = (rs.randn(U, 1) * 0.1).astype(np.float32)
    bi = (rs.randn(I, 1) * 0.1).astype(np.float32)
    batches = [(rs.randint(0, U, B).astype(np.int64), rs.randint(0, I, B).astype(np.int64),
                rs.randint(0, I, B * n_neg).astype(np.int64)) for _ in range(steps)]
    return (Wu, Wi, bu, bi), batches


def make_margin_params(seed, U, I, D):
    """(Wu, Wi, bu, bi) whose hinge margins stay far from the kink: small embeddings (dot products
    of a few hundredths) and item biases on levels 1.5 apart, so that neg - pos + 1 sits near
    1 + {0, +-1.5, +-3} and a step or a few of training cannot carry it to 0."""
    rs = np.random.RandomState(seed)
    Wu = (rs.randn(U, D) * 0.05).astype(np.float32)
    Wi = (rs.randn(I, D) * 0.05).astype(np.float32)
    bu = (rs.randn(U, 1) * 0.1).astype(np.float32)
    bi = (1.5 * rs.randint(0, 3, (I, 1)) + rs.randn(I, 1) * 0.02).astype(np.float32)
    return Wu, Wi, bu, bi


def accumulator_scales(B):
    """Squared typical gradient elements of (Wu, Wi, bu, bi) at make_margin_params' scale for
    one hit in a minibatch of B: score gradients of about 0.2 / B, times a 0.05 row element for
    the embeddings."""
    return [(0.01 / B) ** 2, (0.01 / B) ** 2, (0.2 / B) ** 2, (0.2 / B) ** 2]


def hinge_margin(r):
    """The smallest |neg - pos + 1| of one oracle step: how close the hinge came to its kink."""
    return float(np.abs(r['neg'] - r['pos'] + 1.0).min())


def oracle_run(params, batches, loss, lr, eps=1e-10, n_neg=1, S0=None, each=None):
    """Single-process reference: full-batch oracle step + dense Adagrad (float64).

    ``S0``: initial Adagrad accumulators of (Wu, Wi, bu, bi) instead of zeros; then the final
    accumulators are returned as a third value.  ``each(r)`` sees every step's oracle result."""
    P = [p.astype(np.float64) for p in params]
    S = [np.zeros_like(p) for p in P] if S0 is None else [s.astype(np.float64).reshape(p.shape)
                                                          for s, p in zip(S0, P)]
    losses = []
    for users, items, negs in batches:
        r = omf.mf_step(P[0], P[1], P[2], P[3], users, items, negs, loss, n_neg, np.float64)
        losses.append(float(r['loss']))
        if each is not None:
            each(r)
        for k, g in enumerate((r['dWu'], r['dWi'], r['dbu'], r['dbi'])):
            S[k] += g * g
            P[k] -= lr * g / (np.sqrt(S[k]) + eps)
        del r
    return (P, losses) if S0 is None else (P, losses, S)


def seeded_accumulators(seed, params, scales):
    """Positive Adagrad accumulators for (Wu, Wi, bu, bi): ``scales[k]`` times U[0.5, 1.5], as
    float32.  From a positive start every update is -lr g / sqrt(S0 + g^2), smooth in g, where
    the zero start's first step is lr sign(g) whatever g's magnitude."""
    rs = np.random.RandomState(seed)
    return [(s * rs.uniform(0.5, 1.5, p.shape)).astype(np.float32) for p, s in zip(params, scales)]


def scale_hot_row(S0, table, row, hits):
    """Seeds the accumulators of a row that a minibatch hits ``hits`` times (of embedding table
    ``table`` = 0 for users, 1 for items, and of its bias) at its own gradient scale: its elements
    sum that many terms of random sign.  At the one-hit scale the elements of such a row that
    happen to sum near zero sit in Adagrad's linear regime with a tiny sqrt(S0), which multiplies
    the float32 rounding of their long sums far past that of every other row."""
    S0[table][row] *= hits
    S0[table + 2][row] *= hits


def seed_accumulators(st, S0, pad=1.0):
    """Writes this rank's slices of the full-table accumulators ``S0`` = (Wu, Wi, bu, bi) into a
    ShardState; the padded item rows past the table's end get ``pad``."""
    n = st.ihi - st.ilo
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(st.sWu.device)      # noqa: E731
    st.sWu.copy_(t(S0[0][st.ulo:st.uhi]))
    st.sbu.copy_(t(S0[2].reshape(-1)[st.ulo:st.uhi]))
    st.sWi.fill_(pad)
    st.sbi.fill_(pad)
    st.sWi[:n] = t(S0[1][st.ilo:st.ihi])
    st.sbi[:n] = t(S0[3].reshape(-1)[st.ilo:st.ihi])


def gather_accumulators(st, plan, U, I):
    """The full sWu, sWi, sbu and sbi (biases as columns) of a ShardState on every rank."""
    return [gather_rows(shard, chunk, n) for shard, n, chunk in
            ((st.sWu, U, plan.uchunk), (st.sWi, I, plan.ichunk),
             (st.sbu.reshape(-1, 1), U, plan.uchunk), (st.sbi.reshape(-1, 1), I, plan.ichunk))]


def padded_rows(st):
    """The padded item rows of this rank's shard (past the table's end): W, S, b, sb as NumPy."""
    n = st.ihi - st.ilo
    return [x[n:].cpu().numpy() for x in (st.Wi, st.sWi, st.bi, st.sbi)]


def worst_change(got, ref, start):
    """(index, start, got's change, the oracle's change) of the element where they differ most."""
    start = np.asarray(start, dtype=np.float64).reshape(np.shape(ref))
    d_got = np.asarray(got, dtype=np.float64).reshape(np.shape(ref)) - start
    d_ref = np.asarray(ref, dtype=np.float64) - start
    k = np.unravel_index(np.argmax(np.abs(d_got - d_ref)), d_ref.shape)
    return tuple(int(x) for x in k), float(start[k]), float(d_got[k]), float(d_ref[k])


def change_error(got, ref, start, scale=None):
    """max |(got - start) - (ref - start)| / scale: a table's change against the oracle's, by
    default relative to the oracle's largest change."""
    start = np.asarray(start, dtype=np.float64).reshape(np.shape(ref))
    d_got = np.asarray(got, dtype=np.float64).reshape(np.shape(ref)) - start
    d_ref = np.asarray(ref, dtype=np.float64) - start
    if scale is None:
        scale = np.abs(d_ref).max()
        assert scale > 0, 'the oracle moved nothing'
    return float(np.abs(d_got - d_ref).max() / scale)


TABLE_NAMES = ('Wu', 'Wi', 'bu', 'bi', 'sWu', 'sWi', 'sbu', 'sbi')


def change_errors(got, ref, start, loss, lr):
    """change_error of (Wu, Wi, bu, bi) and their accumulators, by name.  Under bpr and hinge the
    user-bias gradient gp + gn is zero in exact arithmetic, so the oracle moves bu and sbu by
    summation residues only: those two are held relative to one Adagrad step (lr) and to their
    largest starting accumulator instead -- a real gradient there moves them by that much."""
    scales = {}
    if loss in ('bpr', 'hinge'):
        scales = {'bu': lr, 'sbu': float(np.abs(start[6]).max())}
    return {nm: change_error(a, b, s, scales.get(nm)) for a, b, s, nm in zip(got, ref, start, TABLE_NAMES)}


def sharded_run(rank, world, params, batches, loss, lr, device, backend, cache_capacity=None,
                exchange='a2a'):
    """Runs the steps on this rank; returns (all-gathered full tables, losses, exchange stats)."""
    from spotlight_b200.sharded import ShardedMF, ShardPlan, ShardState
    U, D = params[0].shape
    I = params[1].shape[0]
    plan = ShardPlan(U, I, world)
    st = ShardState(plan, rank, D, device, lr=lr, init=[torch.from_numpy(p) for p in params])
    model = ShardedMF(plan, st, rank, backend, cache_capacity=cache_capacity)
    losses = []
    for users, items, negs in batches:
        mine = plan.user_owner(users) == rank
        t = lambda x: torch.from_numpy(x[mine]).to(device)        # noqa: E731
        losses.append(float(model.step(t(users), t(items), t(negs), loss, len(users), exchange)))
    return gather_tables(st, plan, U, I), losses, model.stats


def make_seq_problem(seed, I, D, B, S, steps, layers=0, k=3):
    rs = np.random.RandomState(seed)
    E = (rs.randn(I, D) * 0.3).astype(np.float32)
    E[0] = 0
    bias = (rs.randn(I, 1) * 0.1).astype(np.float32)
    bias[0] = 0
    convs = [((rs.randn(D, D, k, 1) * 0.2).astype(np.float32), (rs.randn(D) * 0.1).astype(np.float32))
             for _ in range(layers)]
    batches = []
    for _ in range(steps):
        seqs = rs.randint(1, I, (B, S)).astype(np.int64)
        for b in range(B):                       # left padding of ragged length, as to_sequence emits
            seqs[b, :rs.randint(0, S)] = 0
        batches.append((seqs, rs.randint(0, I, (B, S)).astype(np.int64)))
    return (E, bias, convs), batches


def seq_oracle_run(params, batches, loss, lr, cnn=None, eps=1e-10):
    """Single-process reference: full-batch oracle sequence step + dense Adagrad (float64)."""
    E, bias, convs = params
    P = [E.astype(np.float64), bias.astype(np.float64)] + [x.astype(np.float64) for wb in convs for x in wb]
    St = [np.zeros_like(p) for p in P]
    losses = []
    for seqs, negs in batches:
        if cnn is None:
            r = oseq.pool_step(P[0], P[1], seqs, negs, loss, 1, np.float64)
            grads = [r['dE'], r['dbias']]
        else:
            cv = [(P[2 + 2 * l], P[3 + 2 * l]) for l in range(len(convs))]
            r = oseq.cnn_step(P[0], P[1], cv, seqs, negs, cnn['kernel_width'], cnn['dilation'], loss, 1,
                              cnn['nonlinearity'], cnn['residual'], np.float64)
            grads = [r['dE'], r['dbias']] + [x for wb in r['dconvs'] for x in wb]
        losses.append(float(r['loss']))
        for k, g in enumerate(grads):
            St[k] += g * g
            P[k] -= lr * g / (np.sqrt(St[k]) + eps)
    return P, losses


def seq_sharded_run(rank, world, params, batches, loss, lr, device, backend, cnn=None):
    """Sequences are dealt round-robin to ranks; returns (gathered E, bias, convs; losses; stats)."""
    from spotlight_b200.sharded import SeqShardState, ShardedSeq, ShardPlan
    E, bias, convs = params
    I, D = E.shape
    plan = ShardPlan(1, I, world)
    st = SeqShardState(plan, rank, D, device, lr=lr, init=(torch.from_numpy(E), torch.from_numpy(bias)),
                       convs=[(torch.from_numpy(w), torch.from_numpy(b)) for w, b in convs])
    model = ShardedSeq(plan, st, rank, backend, cnn=cnn)
    losses = []
    for seqs, negs in batches:
        t = lambda x: torch.from_numpy(np.ascontiguousarray(x[rank::world])).to(device)   # noqa: E731
        losses.append(float(model.step(t(seqs), t(negs), loss)))
    out = [gather_rows(st.Wi, plan.ichunk, I), gather_rows(st.bi.reshape(-1, 1), plan.ichunk, I)]
    out += [x.cpu().numpy() for wb in st.convs for x in wb]
    return out, losses, model.stats


def reference_epochs(seed, users, items, num_items, B, n_iter, n_neg=1):
    """The minibatches the reference loop forms (factorization/implicit.py:114,212-259):
    ctor draw, then per epoch shuffle + one randint per minibatch, all from one stream."""
    rs = np.random.RandomState(seed)
    rs.randint(-10 ** 8, 10 ** 8)
    epochs = []
    for _ in range(n_iter):
        order = np.arange(len(users))
        rs.shuffle(order)
        u, i = users[order], items[order]
        batches = []
        for lo in range(0, len(u), B):
            bu, bi = u[lo:lo + B].astype(np.int64), i[lo:lo + B].astype(np.int64)
            batches.append((bu, bi, rs.randint(0, num_items, len(bu) * n_neg, dtype=np.int64)))
        epochs.append(batches)
    return epochs, rs


def gather_tables(st, plan, U, I):
    """The full Wu, Wi, bu and bi (biases as columns) of a ShardState on every rank."""
    return [gather_rows(shard, chunk, n) for shard, n, chunk in
            ((st.Wu, U, plan.uchunk), (st.Wi, I, plan.ichunk),
             (st.bu.reshape(-1, 1), U, plan.uchunk), (st.bi.reshape(-1, 1), I, plan.ichunk))]


def sharded_fit_run(rank, world, params, users, items, loss, device, backend, seed, B, n_iter, exchange,
                    n_neg=5, S0=None):
    """fit() on this rank; returns (all-gathered full tables, epoch losses, final RandomState).
    With ``S0`` (seed_accumulators) also a fourth value: (all-gathered accumulators, this rank's
    padded item rows)."""
    from spotlight_b200.interactions import Interactions
    from spotlight_b200.sharded import ShardedImplicitFactorizationModel
    U, D = params[0].shape
    I = params[1].shape[0]
    rs = np.random.RandomState(seed)
    model = ShardedImplicitFactorizationModel(U, I, rank, world, device, backend=backend, loss=loss,
                                              embedding_dim=D, n_iter=n_iter, batch_size=B,
                                              learning_rate=0.05, random_state=rs, exchange=exchange,
                                              init=[torch.from_numpy(p) for p in params],
                                              num_negative_samples=n_neg)
    if S0 is not None:
        seed_accumulators(model.state, S0)
    model.fit(Interactions(users, items, num_users=U, num_items=I))
    out = gather_tables(model.state, model.plan, U, I), model.epoch_losses, rs.get_state()
    if S0 is None:
        return out
    return out + ((gather_accumulators(model.state, model.plan, U, I), padded_rows(model.state)),)


# ---------------------------------------------------------------- hashed item table (config 4)

def make_bloom_problem(seed, U, N, M, D, B, steps):
    rs = np.random.RandomState(seed)
    Wu = (rs.randn(U, D) * 0.3).astype(np.float32)
    Wi = (rs.randn(M, D) * 0.3).astype(np.float32)
    Wi[0] = 0
    bu = (rs.randn(U, 1) * 0.1).astype(np.float32)
    bi = (rs.randn(N, 1) * 0.1).astype(np.float32)
    batches = [(rs.randint(0, U, B).astype(np.int64), rs.randint(1, N, B).astype(np.int64),
                rs.randint(0, N, B).astype(np.int64)) for _ in range(steps)]
    return (Wu, Wi, bu, bi), batches


def bloom_oracle_run(params, batches, loss, lr, H, eps=1e-10):
    P = [p.astype(np.float64) for p in params]
    S = [np.zeros_like(p) for p in P]
    losses = []
    for users, items, negs in batches:
        r = omf.mf_bloom_step(P[0], P[1], P[2], P[3], users, items, negs, loss, H, 0, np.float64)
        losses.append(float(r['loss']))
        for k, g in enumerate((r['dWu'], r['dWi'], r['dbu'], r['dbi'])):
            S[k] += g * g
            P[k] -= lr * g / (np.sqrt(S[k]) + eps)
    return P, losses


def bloom_sharded_run(rank, world, params, batches, loss, lr, device, backend, H):
    from spotlight_b200.sharded import BloomShardState, ShardedBloomMF, ShardPlan
    U, D = params[0].shape
    M, N = params[1].shape[0], params[3].shape[0]
    plan = ShardPlan(U, N, world)
    st = BloomShardState(plan, rank, D, device, N, M, H, lr=lr, init=[torch.from_numpy(p) for p in params])
    model = ShardedBloomMF(plan, st, rank, backend)
    losses = []
    for users, items, negs in batches:
        mine = plan.user_owner(users) == rank
        t = lambda x: torch.from_numpy(x[mine]).to(device)        # noqa: E731
        losses.append(float(model.step(t(users), t(items), t(negs), loss, len(users))))
    out = [gather_rows(shard, chunk, n) for shard, n, chunk in
           ((st.Wu, U, plan.uchunk), (st.Wi, M, st.mchunk), (st.bu.reshape(-1, 1), U, plan.uchunk))]
    out.append(st.bi.reshape(-1, 1).cpu().numpy())           # replicated
    return out, losses

