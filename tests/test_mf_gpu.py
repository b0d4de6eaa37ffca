"""GPU parity tests for the matrix-factorisation hot path: the CUDA kernels
(reached through the C-ABI) against the committed golden vectors of the live
reference, against the oracle on seeded inputs, and -- at benchmark sizes --
through size-independent properties (bit-reproducibility, conservation sums,
agreement with an fp32 ATen restatement).

Tolerance: integer work (sampling, hashing, row indexing) bit-exact; floating
point 1e-5 relative to the tensor's max magnitude (north star).
"""

import numpy as np
import pytest
import torch

from conftest import assert_close, load_golden
from oracle import mf as omf

pytestmark = pytest.mark.gpu

LOSS_OF = {'mf_pointwise': 'pointwise', 'mf_bpr': 'bpr', 'mf_hinge': 'hinge',
           'mf_adaptive_hinge': 'adaptive_hinge', 'mf_bpr_d64': 'bpr'}


def dev():
    return torch.device('cuda:0')


def t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(dev())


def assert_close_dev(actual, expected, rtol=1e-5, atol=0.0, what=''):
    """conftest.assert_close for multi-GB tensors: same criterion, evaluated on the device."""
    assert actual.shape == expected.shape, (what, actual.shape, expected.shape)
    scale = expected.abs().max().item()
    err = (actual - expected).abs().max().item()
    tol = rtol * scale + atol
    assert err <= tol, '%s: max err %.3e > tol %.3e (scale %.3e)' % (what, err, tol, scale)


# ------------------------------------------------------------------ sampler

@pytest.mark.parametrize('num_items,shape', [(100000, 70000), (1683, (5, 77)), (1000000, 1234),
                                             (50000000, 999), (1, 5), (2, 7), (4096, 3000),
                                             (4097, 3000), (100000, 1), (100000, 2_000_003)])
def test_sampler_bit_exact(num_items, shape):
    from spotlight_b200.sampling import sample_items
    a, b = np.random.RandomState(123), np.random.RandomState(123)
    a.randint(0, 10, 77)
    b.randint(0, 10, 77)          # start mid-block
    want = a.randint(0, num_items, shape, dtype=np.int64)
    got = sample_items(num_items, shape, random_state=b, device=dev())
    assert got.dtype == torch.int64 and tuple(got.shape) == want.shape
    assert (got.cpu().numpy() == want).all()
    sa, sb = a.get_state(), b.get_state()
    assert (sa[1] == sb[1]).all() and sa[2] == sb[2]
    # and the stream continues identically on the host
    assert (a.randint(0, 1000, 50) == b.randint(0, 1000, 50)).all()


def test_parallel_generator_matches_sequential_and_numpy():
    """Jump-ahead (GF(2) polynomial) block generation: bit-identical to the
    single-CTA generator and to NumPy on a 30 M-value draw (config-2 epoch scale)."""
    import ctypes
    from spotlight_b200 import _lib, rng
    from spotlight_b200.ops import _ptr, _stream
    lib = _lib.load()
    key = np.random.RandomState(11).get_state()[1]
    for nblocks in (4097, 20000, 70001):
        a = torch.zeros(nblocks * 624, dtype=torch.int32, device=dev())
        b = torch.zeros_like(a)
        a[:624] = torch.from_numpy(key.view(np.int32)).to(dev())
        b[:624] = a[:624]
        _lib.check(lib.slb_mt19937_fill(_ptr(a), nblocks, _stream()), 'seq')
        table, rows, direct, drows = rng._jump_table(dev())
        states = rng._states(dev(), 4096)
        _lib.check(lib.slb_mt19937_fill_parallel(_ptr(b), nblocks, _ptr(table), rows, _ptr(states),
                                                 _stream()), 'par')
        assert torch.equal(a, b), nblocks
        # one-round generator: precomputed multiples of 256 blocks (+ doubling over the coarse
        # slots once the stream exceeds 256 fine slots: 70001 blocks = 274 slots)
        c = torch.zeros_like(a)
        c[:624] = a[:624]
        _lib.check(lib.slb_mt19937_fill_direct(_ptr(c), nblocks, _ptr(table), rows, _ptr(direct), drows,
                                               rng._J0_LOG2, _ptr(states), states.numel() // 624,
                                               _stream()), 'direct')
        assert torch.equal(a, c), nblocks
    from spotlight_b200.sampling import sample_items
    r1, r2 = np.random.RandomState(5), np.random.RandomState(5)
    want = r1.randint(0, 100000, 30_000_000, dtype=np.int64)
    got = sample_items(100000, 30_000_000, random_state=r2, device=dev())
    assert (got.cpu().numpy() == want).all()
    s1, s2 = r1.get_state(), r2.get_state()
    assert (s1[1] == s2[1]).all() and s1[2] == s2[2]


def test_chained_draws_one_sync():
    """DeviceStream: many draws (one per minibatch in the reference, implicit.py:256-259)
    chained on the device, one hand-back at the end -- bit-exact values and final state."""
    from spotlight_b200.rng import DeviceStream
    a, b = np.random.RandomState(77), np.random.RandomState(77)
    a.randint(0, 10, 300); b.randint(0, 10, 300)
    plan = [(100000, 524288), (100000, 1), (1683, 4097), (100000, 3_000_000), (50000000, 70000),
            (1, 9), (100000, 624), (1000000, 2_500_000)]
    want = [a.randint(0, n, c, dtype=np.int64) for n, c in plan]
    with torch.cuda.stream(torch.cuda.Stream()):
        st = DeviceStream(b, dev())
        got = [st.draw(n, c) for n, c in plan]
        st.finish()
    for w, g, pc in zip(want, got, plan):
        assert (g.cpu().numpy() == w).all(), pc
    sa, sb = a.get_state(), b.get_state()
    assert (sa[1] == sb[1]).all() and sa[2] == sb[2]
    assert (a.randint(0, 1000, 50) == b.randint(0, 1000, 50)).all()
    # gaussian cache of the RandomState survives the take-over (ADVICE r1)
    c = np.random.RandomState(3)
    c.standard_normal(1)
    has, val = c.get_state()[3:5]
    st = DeviceStream(c, dev())
    st.draw(1000, 10)
    st.finish()
    assert c.get_state()[3:5] == (has, val)


def test_sampler_golden_stream():
    from spotlight_b200.sampling import sample_items
    g = load_golden('rng_stream')
    rs = np.random.RandomState(42)
    assert rs.randint(-10**8, 10**8) == int(g['ctor'])
    idx = np.arange(1000)
    rs.shuffle(idx)
    for key, (n, sz) in zip(['n0', 'n1', 'n2', 'n3', 'n4'],
                            [(100000, 257), (1683, 64), (1000000, 100), (50000000, 33),
                             (1683, (5, 7))]):
        got = sample_items(n, sz, random_state=rs, device=dev())
        assert (got.cpu().numpy() == g[key]).all(), key
    st = rs.get_state()
    assert (st[1] == g['end_key']).all() and st[2] == int(g['end_pos'])


# --------------------------------------------------------------- fused step

def _params(g):
    return (t(g['sd.user_embeddings.weight']), t(g['sd.item_embeddings.weight']),
            t(g['sd.user_biases.weight']), t(g['sd.item_biases.weight']))


@pytest.mark.parametrize('name', sorted(LOSS_OF))
def test_fused_step_golden(name):
    from spotlight_b200 import ops
    from spotlight_b200._lib import LOSS_KIND
    g = load_golden(name)
    loss = LOSS_OF[name]
    n_neg = int(g['n_neg']) if loss == 'adaptive_hinge' else 1
    Wu, Wi, bu, bi = _params(g)
    out = ops.mf_train_step(Wu, Wi, bu, bi, t(g['users']), t(g['items']), t(g['negs']),
                            LOSS_KIND[loss], n_neg, True)
    l, pos, neg, dWu, dWi, dbu, dbi = [o.cpu().numpy() for o in out]
    assert_close(pos, g['pos'], 1e-5, what='pos')
    assert_close(neg.reshape(g['neg'].shape), g['neg'], 1e-5, what='neg')
    assert_close(l, g['loss'], 1e-5, what='loss')
    assert_close(dWu, g['grad.user_embeddings.weight'], 1e-5, what='dWu')
    assert_close(dWi, g['grad.item_embeddings.weight'], 1e-5, what='dWi')
    assert_close(dbu, g['grad.user_biases.weight'], 1e-5, atol=1e-7, what='dbu')
    assert_close(dbi, g['grad.item_biases.weight'], 1e-5, what='dbi')
    # untouched rows are exactly zero, like the reference's dense grad
    ref_zero = np.abs(g['grad.item_embeddings.weight']).sum(1) == 0
    assert np.all(dWi[ref_zero] == 0)


@pytest.mark.parametrize('loss', ['pointwise', 'bpr', 'hinge', 'adaptive_hinge'])
@pytest.mark.parametrize('dim', [4, 8, 24, 128, 256])
def test_fused_step_vs_oracle_dims(loss, dim):
    from spotlight_b200 import ops
    from spotlight_b200._lib import LOSS_KIND
    rs = np.random.RandomState(dim)
    U, I, B, n_neg = 211, 97, 777, (3 if loss == 'adaptive_hinge' else 1)
    Wu = (rs.randn(U, dim) * 0.3).astype(np.float32)
    Wi = (rs.randn(I, dim) * 0.3).astype(np.float32)
    bu = (rs.randn(U, 1) * 0.1).astype(np.float32)
    bi = (rs.randn(I, 1) * 0.1).astype(np.float32)
    users = rs.randint(0, U, B).astype(np.int64)
    items = rs.randint(0, I, B).astype(np.int64)
    negs = rs.randint(0, I, B * n_neg).astype(np.int64)
    ref = omf.mf_step(Wu, Wi, bu, bi, users, items, negs, loss, n_neg, np.float64)
    out = ops.mf_train_step(t(Wu), t(Wi), t(bu), t(bi), t(users), t(items), t(negs),
                            LOSS_KIND[loss], n_neg, True)
    l, pos, neg, dWu, dWi, dbu, dbi = [o.cpu().numpy() for o in out]
    assert_close(pos, ref['pos'], 1e-5, what='pos')
    assert_close(neg.reshape(ref['neg'].shape), ref['neg'], 1e-5, what='neg')
    assert_close(l, ref['loss'], 1e-5, what='loss')
    assert_close(dWu, ref['dWu'], 1e-5, what='dWu')
    assert_close(dWi, ref['dWi'], 1e-5, what='dWi')
    assert_close(dbu, ref['dbu'], 1e-5, atol=1e-7, what='dbu')
    assert_close(dbi, ref['dbi'], 1e-5, what='dbi')


def test_fused_step_hot_rows_and_batch_of_one():
    """Heavy duplication (every interaction hits the same few rows: the
    long-segment path) and the batch-of-one case the reference cannot run."""
    from spotlight_b200 import ops
    rs = np.random.RandomState(1)
    U, I, D, B = 5, 3, 32, 4000
    Wu = (rs.randn(U, D) * 0.3).astype(np.float32)
    Wi = (rs.randn(I, D) * 0.3).astype(np.float32)
    bu = np.zeros((U, 1), np.float32)
    bi = np.zeros((I, 1), np.float32)
    users = rs.randint(0, U, B).astype(np.int64)
    items = rs.randint(0, I, B).astype(np.int64)
    negs = rs.randint(0, I, B).astype(np.int64)
    ref = omf.mf_step(Wu, Wi, bu, bi, users, items, negs, 'bpr', 1, np.float64)
    out = ops.mf_train_step(t(Wu), t(Wi), t(bu), t(bi), t(users), t(items), t(negs), 1, 1, False)
    assert_close(out[3].cpu().numpy(), ref['dWu'], 1e-5, what='dWu hot')
    assert_close(out[4].cpu().numpy(), ref['dWi'], 1e-5, what='dWi hot')
    ref1 = omf.mf_step(Wu, Wi, bu, bi, users[:1], items[:1], negs[:1], 'hinge', 1, np.float64)
    out1 = ops.mf_train_step(t(Wu), t(Wi), t(bu), t(bi), t(users[:1]), t(items[:1]), t(negs[:1]),
                             2, 1, False)
    assert_close(out1[0].cpu().numpy(), ref1['loss'], 1e-5, what='loss b1')
    assert_close(out1[3].cpu().numpy(), ref1['dWu'], 1e-5, what='dWu b1')


def test_fused_step_zipf_hot_rows():
    """Skewed item popularity (Zipf) at a large batch: the hottest item owns tens of
    thousands of terms.  Hot rows are sorted by the bitmap kernel and must stay
    correct (vs an fp32 ATen restatement), bit-reproducible and reasonably fast."""
    import time
    from spotlight_b200 import ops
    torch.manual_seed(1)
    U, I, D, B = 200_000, 20_000, 64, 262_144
    d = dev()
    Wu = torch.randn(U, D, device=d) / D
    Wi = torch.randn(I, D, device=d) / D
    bu = torch.zeros(U, 1, device=d)
    bi = torch.zeros(I, 1, device=d)
    p = 1.0 / torch.arange(1, I + 1, device=d, dtype=torch.float64)
    items = torch.multinomial(p / p.sum(), B, replacement=True)
    users = torch.randint(0, U, (B,), device=d)
    negs = torch.randint(0, I, (B,), device=d)
    hottest = int(torch.bincount(items).max())
    assert hottest > 10_000
    o1 = ops.mf_train_step(Wu, Wi, bu, bi, users, items, negs, 1, 1, False)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    o2 = ops.mf_train_step(Wu, Wi, bu, bi, users, items, negs, 1, 1, False)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    assert torch.equal(o1[4], o2[4]) and torch.equal(o1[3], o2[3])
    u, qi, qj = Wu[users], Wi[items], Wi[negs]
    s = torch.sigmoid((u * qi).sum(1) - (u * qj).sum(1))
    gp = -(s * (1 - s)) / B
    rWi = torch.zeros_like(Wi).index_add_(0, items, gp[:, None] * u).index_add_(0, negs, -gp[:, None] * u)
    assert_close(o1[4].cpu().numpy(), rWi.cpu().numpy(), 5e-5, what='dWi zipf')
    assert dt < 0.5, 'hot-row path too slow: %.3f s (hottest item %d terms)' % (dt, hottest)


def test_fused_step_full_size_properties():
    """BASELINE config 2 shape (1M users x 100K items x 64, B = 65536):
    bit-reproducible, conservation identities, and agreement with an fp32 ATen
    restatement of the same step."""
    from spotlight_b200 import ops
    torch.manual_seed(0)
    U, I, D, B = 1_000_000, 100_000, 64, 65536
    d = dev()
    Wu = torch.randn(U, D, device=d) / D
    Wi = torch.randn(I, D, device=d) / D
    bu = torch.randn(U, 1, device=d) * 0.01
    bi = torch.randn(I, 1, device=d) * 0.01
    users = torch.randint(0, U, (B,), device=d)
    items = torch.randint(0, I, (B,), device=d)
    negs = torch.randint(0, I, (B,), device=d)
    o1 = ops.mf_train_step(Wu, Wi, bu, bi, users, items, negs, 1, 1, True)
    o2 = ops.mf_train_step(Wu, Wi, bu, bi, users, items, negs, 1, 1, True)
    for a, b in zip(o1, o2):
        assert torch.equal(a, b), 'fused step is not bit-reproducible'
    loss, pos, neg, dWu, dWi, dbu, dbi = o1
    # ATen fp32 restatement
    u, qi, qj = Wu[users], Wi[items], Wi[negs]
    p = (u * qi).sum(1) + bu[users, 0] + bi[items, 0]
    n = (u * qj).sum(1) + bu[users, 0] + bi[negs, 0]
    s = torch.sigmoid(p - n)
    assert_close(pos.cpu().numpy(), p.cpu().numpy(), 1e-5, what='pos')
    assert_close(loss.item(), (1 - s).mean().item(), 1e-5, what='loss')
    gp = -(s * (1 - s)) / B
    rWu = torch.zeros_like(Wu).index_add_(0, users, gp[:, None] * (qi - qj))
    rWi = torch.zeros_like(Wi).index_add_(0, items, gp[:, None] * u).index_add_(0, negs, -gp[:, None] * u)
    assert_close(dWu.cpu().numpy(), rWu.cpu().numpy(), 1e-5, what='dWu')
    assert_close(dWi.cpu().numpy(), rWi.cpu().numpy(), 2e-5, what='dWi')
    # conservation: bpr gives gp + gn = 0 per interaction
    assert abs(dbi.double().sum().item()) < 1e-6
    assert torch.count_nonzero(dbu).item() == 0 or dbu.abs().max().item() < 1e-9


# ------------------------------------------------- planned two-kernel step
# (against the float64 oracle: tests/test_mf_planned_oracle_gpu.py)

@pytest.mark.parametrize('opt', ['sgd', 'adagrad'])
def test_planned_step_equals_first_generation(opt):
    """Same minibatches through the planned step and through the first-generation
    (forward / index / backward / apply) step: three steps, Zipf-skewed items so that hot item
    rows take the long-list kernels on both paths."""
    from spotlight_b200 import _lib, ops
    torch.manual_seed(5)
    U, I, D, B = 50_000, 20_000, 64, 200_000
    d = dev()
    base = [torch.randn(U, D, device=d) / D, torch.randn(I, D, device=d) / D,
            torch.randn(U, 1, device=d) * 0.01, torch.randn(I, 1, device=d) * 0.01]
    pz = 1.0 / torch.arange(1, I + 1, device=d, dtype=torch.float64)
    batches = [(torch.randint(0, U, (B,), device=d), torch.multinomial(pz / pz.sum(), B, replacement=True),
                torch.randint(0, I, (B,), device=d)) for _ in range(3)]
    batches[1][0][:5000] = 17                     # a hot *user* row too (5000 interactions in one batch)
    assert int(torch.bincount(batches[0][1]).max()) > 5000
    kind = _lib.OPT_SGD if opt == 'sgd' else _lib.OPT_ADAGRAD
    res = {}
    for planned in (True, False):
        prm = [x.clone() for x in base]
        states = [torch.zeros_like(x) for x in prm]
        losses = [ops.mf_train_step_inplace(*prm, u, i, j, 'bpr', kind, 0.5 if opt == 'sgd' else 0.05,
                                            states=states, planned=planned).item() for u, i, j in batches]
        res[planned] = (prm, losses)
    assert_close(np.array(res[True][1]), np.array(res[False][1]), 1e-6, what='losses')
    for a, b, nm in zip(res[True][0], res[False][0], ('Wu', 'Wi', 'bu', 'bi')):
        # two correct fp32 summation orders; Adagrad's first-touch normalisation amplifies them
        assert_close_dev(a, b, 1e-5 if opt == 'sgd' else 5e-3, what=nm)


def test_planned_epoch_full_size_two_streams():
    """BASELINE config 2 shape through slb_mf_fit_epoch (plan on its own stream, double
    buffered): 6 steps of B = 524288 equal the same steps issued one by one on one stream."""
    import ctypes
    from spotlight_b200 import _lib, ops
    torch.manual_seed(6)
    U, I, D, B, K = 1_000_000, 100_000, 64, 524_288, 6
    d = dev()
    base = [torch.randn(U, D, device=d) / D, torch.randn(I, D, device=d) / D,
            torch.zeros(U, 1, device=d), torch.zeros(I, 1, device=d)]
    users = torch.randint(0, U, (K * B - 1000,), device=d)          # short last batch
    items = torch.randint(0, I, (K * B - 1000,), device=d)
    negs = torch.randint(0, I, (K * B - 1000,), device=d)
    lib = _lib.load()
    # one by one
    p1 = [x.clone() for x in base]
    s1 = [torch.zeros_like(x) for x in p1]
    l1 = []
    for k in range(K):
        sl = slice(k * B, min((k + 1) * B, users.numel()))
        l1.append(ops.mf_train_step_inplace(*p1, users[sl], items[sl], negs[sl], 'bpr', _lib.OPT_ADAGRAD,
                                            0.05, states=s1).item())
    # one C call, plan stream
    p2 = [x.clone() for x in base]
    s2 = [torch.zeros_like(x) for x in p2]
    a = ops.mf_step_args(*p2, users, items, negs, 'bpr', 1, batch=B)
    a.grad_mode = _lib.GRAD_COMPACT
    a.opt, a.lr, a.weight_decay, a.eps = _lib.OPT_ADAGRAD, 0.05, 0.0, 1e-10
    a.state_Wu, a.state_Wi, a.state_bu, a.state_bi = [x.data_ptr() for x in s2]
    fws = ops.workspace('mfv2_%d_%d_%d' % (U, I, D), lib.slb_mf_fused_workspace_bytes(B, U, I, D), d)
    a.fused_workspace, a.fused_workspace_bytes = fws.data_ptr(), fws.numel()
    ws = ops.workspace('mf%d_%d' % (U, I), lib.slb_mf_step_workspace_bytes(B, 1, 1, U, I), d)
    a.workspace, a.workspace_bytes = ws.data_ptr(), ws.numel()
    plan = torch.cuda.Stream()
    a.plan_stream = plan.cuda_stream
    losses = torch.empty(K, device=d)
    _lib.check(lib.slb_mf_fit_epoch(ctypes.byref(a), ops._ptr(users), ops._ptr(items), ops._ptr(negs),
                                    users.numel(), ops._ptr(losses), ops._stream()), 'fit_epoch')
    torch.cuda.synchronize()
    assert_close(losses.cpu().numpy(), np.array(l1), 1e-7, what='losses')
    for x, y in zip(p1 + s1, p2 + s2):
        assert torch.equal(x, y), 'two-stream epoch differs from step-by-step'
    assert not ops.workspace_error_flag(ws)


def test_fused_step_config3_size():
    """BASELINE config 3 shape on one GPU (10M users x 1M items x 128, adaptive hinge with
    n = 5 negatives, B = 65536): loss, scores and all gradients vs an fp32 ATen restatement
    of the reference step *including* its user/negative pairing (implicit.py:266-275: flat
    negative f is scored with users[f // n] and read as element (f // B, f % B))."""
    from spotlight_b200 import ops
    torch.manual_seed(3)
    U, I, D, B, n = 10_000_000, 1_000_000, 128, 65536, 5
    d = dev()
    Wu = torch.randn(U, D, device=d) / D
    Wi = torch.randn(I, D, device=d) / D
    bu = torch.randn(U, 1, device=d) * 0.01
    bi = torch.randn(I, 1, device=d) * 0.01
    users = torch.randint(0, U, (B,), device=d)
    items = torch.randint(0, I, (B,), device=d)
    negs = torch.randint(0, I, (B * n,), device=d)
    loss, pos, neg, dWu, dWi, dbu, dbi = ops.mf_train_step(Wu, Wi, bu, bi, users, items, negs, 3, n, True)
    u_rep = users.view(B, 1).expand(B, n).reshape(B * n)
    p = (Wu[users] * Wi[items]).sum(1) + bu[users, 0] + bi[items, 0]
    s = (Wu[u_rep] * Wi[negs]).sum(1) + bu[u_rep, 0] + bi[negs, 0]
    hardest, k = s.view(n, B).max(0)
    z = hardest - p + 1.0
    assert_close(pos.cpu().numpy(), p.cpu().numpy(), 1e-5, what='pos')
    assert_close(neg.cpu().numpy(), s.cpu().numpy(), 1e-5, what='neg')
    assert_close(loss.item(), z.clamp(min=0).mean().item(), 1e-5, what='loss')
    act = (z >= 0).float() / B
    f = k * B + torch.arange(B, device=d)                   # flat index of the arg-max negative
    rWu = torch.zeros_like(Wu).index_add_(0, users, -act[:, None] * Wi[items])
    rWu.index_add_(0, u_rep[f], act[:, None] * Wi[negs[f]])
    assert_close_dev(dWu, rWu, 1e-5, what='dWu')
    del rWu
    rWi = torch.zeros_like(Wi).index_add_(0, items, -act[:, None] * Wu[users])
    rWi.index_add_(0, negs[f], act[:, None] * Wu[u_rep[f]])
    assert_close_dev(dWi, rWi, 1e-5, what='dWi')
    rbu = torch.zeros(U, device=d).index_add_(0, users, -act).index_add_(0, u_rep[f], act)
    rbi = torch.zeros(I, device=d).index_add_(0, items, -act).index_add_(0, negs[f], act)
    assert_close_dev(dbu.reshape(-1), rbu, 1e-5, atol=1e-9, what='dbu')
    assert_close_dev(dbi.reshape(-1), rbi, 1e-5, atol=1e-9, what='dbi')
    o2 = ops.mf_train_step(Wu, Wi, bu, bi, users, items, negs, 3, n, False)
    assert torch.equal(o2[3], dWu) and torch.equal(o2[4], dWi), 'not bit-reproducible'


def test_fused_bloom_step_config4_size():
    """BASELINE config 4 shape on one GPU (BloomEmbedding 50M items -> 1M hashed rows, D = 64,
    H = 4, hinge, plain 1M-user table, item bias unhashed 50M x 1, B = 65536): the fused
    hashed step vs an fp32 ATen restatement built on the oracle's murmur rows
    (layers.py:178-204, 240-241)."""
    from oracle.murmur import bloom_rows
    from spotlight_b200 import ops
    from spotlight_b200.layers import SEEDS
    torch.manual_seed(4)
    U, N, M, D, H, B = 1_000_000, 50_000_000, 1_000_000, 64, 4, 65536
    d = dev()
    Wu = torch.randn(U, D, device=d) / D
    Wi = torch.randn(M, D, device=d) / D
    Wi[0] = 0                                                # padding row of the hashed table
    bu = torch.randn(U, 1, device=d) * 0.01
    bi = torch.randn(N, 1, device=d) * 0.01
    rs = np.random.RandomState(44)
    users = t(rs.randint(0, U, B).astype(np.int64))
    items_h = rs.randint(1, N, B).astype(np.int64)
    negs_h = rs.randint(0, N, B).astype(np.int64)
    negs_h[:3] = 0                                           # the padding id among the negatives
    items, negs = t(items_h), t(negs_h)
    loss, pos, neg, dWu, dWi, dbu, dbi = ops.mf_bloom_train_step(Wu, Wi, bu, bi, users, items, negs, 2, 1,
                                                                [], SEEDS[:H], -1, 0, True)
    ri, rj = t(bloom_rows(items_h, H, M)), t(bloom_rows(negs_h, H, M))      # (B, H) int64, oracle murmur
    assert int(rj[:3].abs().sum()) == 0
    u = Wu[users]
    qi, qj = Wi[ri].sum(1), Wi[rj].sum(1)
    p = (u * qi).sum(1) + bu[users, 0] + bi[items, 0]
    ng = (u * qj).sum(1) + bu[users, 0] + bi[negs, 0]
    z = ng - p + 1.0
    assert_close(pos.cpu().numpy(), p.cpu().numpy(), 1e-5, what='pos')
    assert_close(neg.cpu().numpy(), ng.cpu().numpy(), 1e-5, what='neg')
    assert_close(loss.item(), z.clamp(min=0).mean().item(), 1e-5, what='loss')
    act = (z >= 0).float() / B
    rWu = torch.zeros_like(Wu).index_add_(0, users, act[:, None] * (qj - qi))
    gu = act[:, None] * u
    rWi = torch.zeros_like(Wi)
    for k in range(H):
        rWi.index_add_(0, ri[:, k], -gu).index_add_(0, rj[:, k], gu)
    rWi[0] = 0                                               # frozen padding row
    assert_close_dev(dWu, rWu, 1e-5, what='dWu')
    assert_close_dev(dWi, rWi, 1e-5, what='dWi')
    rbi = torch.zeros(N, device=d).index_add_(0, items, -act).index_add_(0, negs, act)
    assert_close_dev(dbi.reshape(-1), rbi, 1e-5, atol=1e-9, what='dbi')
    assert dbu.abs().max().item() < 1e-9                     # hinge: gp + gn = 0 per interaction


# -------------------------------------------------------- scores / embedding

def test_mf_scores_forward_backward_vs_autograd():
    from spotlight_b200 import ops
    rs = np.random.RandomState(4)
    U, I, D, B = 50, 40, 32, 300
    Wu = t((rs.randn(U, D) * 0.3).astype(np.float32)).requires_grad_()
    Wi = t((rs.randn(I, D) * 0.3).astype(np.float32)).requires_grad_()
    bu = t((rs.randn(U, 1) * 0.1).astype(np.float32)).requires_grad_()
    bi = t((rs.randn(I, 1) * 0.1).astype(np.float32)).requires_grad_()
    users = t(rs.randint(0, U, B).astype(np.int64))
    items = t(rs.randint(0, I, B).astype(np.int64))
    w = t(rs.randn(B).astype(np.float32))
    (ops.mf_scores(Wu, Wi, bu, bi, users, items) * w).sum().backward()
    got = [p.grad.clone() for p in (Wu, Wi, bu, bi)]
    for p in (Wu, Wi, bu, bi):
        p.grad = None
    ref = (Wu[users] * Wi[items]).sum(1) + bu[users, 0] + bi[items, 0]
    (ref * w).sum().backward()
    for a, p, nm in zip(got, (Wu, Wi, bu, bi), 'Wu Wi bu bi'.split()):
        assert_close(a.cpu().numpy(), p.grad.cpu().numpy(), 1e-5, what=nm)
    # one user broadcast over all items (predict path)
    one = ops.mf_scores(Wu, Wi, bu, bi, users[:1], torch.arange(I, device=dev()))
    ref1 = (Wu[users[:1]] * Wi).sum(1) + bu[users[0], 0] + bi[:, 0]
    assert_close(one.detach().cpu().numpy(), ref1.detach().cpu().numpy(), 1e-5, what='bcast')


@pytest.mark.parametrize('name', ['mf_hinge_bloom', 'mf_adaptive_bloom'])
def test_bloom_rows_bit_exact(name):
    from spotlight_b200.layers import BloomEmbedding
    g = load_golden(name)
    layer = BloomEmbedding(int(g['num_items']), int(g['dim']),
                           compression_ratio=float(g['bloom_ratio']),
                           num_hash_functions=int(g['bloom_H'])).to(dev())
    rows = layer._get_hashed_indices(t(g['items'])).cpu().numpy()
    assert (rows == g['bloom_rows_items']).all()
    big = np.random.RandomState(0).randint(0, 50_000_000, 20000).astype(np.int64)
    big[:3] = [0, 49_999_999, 2**31 - 1]
    from spotlight_b200 import ops
    from oracle.murmur import bloom_rows, SEEDS
    got = ops.bloom_rows(t(big), SEEDS[:4], 1_000_000, 0).cpu().numpy()
    assert (got == bloom_rows(big, 4, 1_000_000)).all()


@pytest.mark.parametrize('name,loss', [('mf_hinge_bloom', 'hinge'),
                                       ('mf_adaptive_bloom', 'adaptive_hinge')])
def test_generic_route_bloom_golden(name, loss):
    """BilinearNet with a BloomEmbedding item layer through the generic
    (gather op + loss op + autograd) route vs the reference's grads."""
    from spotlight_b200.factorization.representations import BilinearNet
    from spotlight_b200.layers import BloomEmbedding, ScaledEmbedding
    from spotlight_b200 import losses
    g = load_golden(name)
    U, I, D = int(g['num_users']), int(g['num_items']), int(g['dim'])
    net = BilinearNet(U, I, D, user_embedding_layer=ScaledEmbedding(U, D),
                      item_embedding_layer=BloomEmbedding(
                          I, D, compression_ratio=float(g['bloom_ratio']),
                          num_hash_functions=int(g['bloom_H'])))
    net.load_state_dict({k[3:]: torch.from_numpy(v) for k, v in g.items() if k.startswith('sd.')})
    net = net.to(dev())
    users, items, negs = t(g['users']), t(g['items']), t(g['negs'])
    B = users.numel()
    pos = net(users, items)
    if loss == 'adaptive_hinge':
        n = int(g['n_neg'])
        rep = users.view(B, 1).expand(B, n).reshape(B * n)
        neg = net(rep, negs).view(n, B)
        l = losses.adaptive_hinge_loss(pos, neg)
    else:
        neg = net(users, negs)
        l = losses.hinge_loss(pos, neg)
    l.backward()
    assert_close(pos.detach().cpu().numpy(), g['pos'], 1e-5, what='pos')
    assert_close(neg.detach().cpu().numpy(), g['neg'], 1e-5, what='neg')
    assert_close(l.item(), g['loss'], 1e-5, what='loss')
    for k, p in net.named_parameters():
        assert_close(p.grad.cpu().numpy(), g['grad.' + k], 1e-5, atol=1e-7, what=k)


@pytest.mark.parametrize('name,loss', [('mf_hinge_bloom', 'hinge'),
                                       ('mf_adaptive_bloom', 'adaptive_hinge')])
def test_fused_bloom_step_golden(name, loss):
    """The fused hashed-table step (one forward kernel with in-register murmur3, the
    common deterministic backward, scalar bias scatter) vs the reference's grads."""
    from spotlight_b200 import ops
    from spotlight_b200._lib import LOSS_KIND
    from spotlight_b200.layers import SEEDS
    g = load_golden(name)
    H = int(g['bloom_H'])
    n_neg = int(g['n_neg']) if loss == 'adaptive_hinge' else 1
    out = ops.mf_bloom_train_step(t(g['sd.user_embeddings.weight']),
                                  t(g['sd.item_embeddings.embeddings.weight']),
                                  t(g['sd.user_biases.weight']), t(g['sd.item_biases.weight']),
                                  t(g['users']), t(g['items']), t(g['negs']), LOSS_KIND[loss], n_neg,
                                  [], SEEDS[:H], -1, 0, True)
    l, pos, neg, dWu, dWi, dbu, dbi = [o.cpu().numpy() for o in out]
    assert_close(pos, g['pos'], 1e-5, what='pos')
    assert_close(neg.reshape(g['neg'].shape), g['neg'], 1e-5, what='neg')
    assert_close(l, g['loss'], 1e-5, what='loss')
    assert_close(dWu, g['grad.user_embeddings.weight'], 1e-5, what='dWu')
    assert_close(dWi, g['grad.item_embeddings.embeddings.weight'], 1e-5, what='dWi')
    assert_close(dbu, g['grad.user_biases.weight'], 1e-5, atol=1e-7, what='dbu')
    assert_close(dbi, g['grad.item_biases.weight'], 1e-5, what='dbi')
    assert np.all(dWi[0] == 0)          # the padding row of the compressed table is frozen


@pytest.mark.parametrize('name,loss', [('mf_hinge_bloom', 'hinge'), ('mf_adaptive_bloom', 'adaptive_hinge')])
def test_fused_bloom_inplace_sgd_golden(name, loss):
    """Hashed-table step with the optimizer fused in (compact row gradients, hash-bucket sparse
    bias update, nothing dense): one SGD step reproduces W - lr * (the live reference's gradient)."""
    from spotlight_b200 import _lib, ops
    from spotlight_b200.layers import SEEDS
    g = load_golden(name)
    H = int(g['bloom_H'])
    n_neg = int(g['n_neg']) if loss == 'adaptive_hinge' else 1
    names = ['user_embeddings.weight', 'item_embeddings.embeddings.weight', 'user_biases.weight', 'item_biases.weight']
    grads = [g['grad.' + k] for k in names]
    lr = 0.3 / max(np.abs(x).max() for x in grads[:2])
    prm = [t(g['sd.' + k].copy()) for k in names]
    l = ops.mf_bloom_train_step_inplace(*prm, t(g['users']), t(g['items']), t(g['negs']), loss, n_neg,
                                        [], SEEDS[:H], -1, 0, _lib.OPT_SGD, lr)
    assert_close(l.item(), g['loss'], 1e-5, what='loss')
    for k, p, gr in zip(names, prm, grads):
        want = g['sd.' + k].astype(np.float64) - lr * gr
        assert_close(p.cpu().numpy(), want, 5e-6, what=k)


def test_fused_bloom_config4_inplace_vs_dense():
    """BASELINE config 4 shape: the in-place fused step equals the dense-gradient step followed by
    the same optimizer (SGD tables; Adagrad accumulators = g^2), including the 50 M-row item bias."""
    from spotlight_b200 import _lib, ops
    from spotlight_b200.layers import SEEDS
    torch.manual_seed(4)
    U, N, M, D, H, B = 1_000_000, 50_000_000, 1_000_000, 64, 4, 65536
    d = dev()
    base = [torch.randn(U, D, device=d) / D, torch.randn(M, D, device=d) / D,
            torch.randn(U, 1, device=d) * 0.01, torch.randn(N, 1, device=d) * 0.01]
    base[1][0] = 0
    rs = np.random.RandomState(45)
    users, items, negs = t(rs.randint(0, U, B).astype(np.int64)), t(rs.randint(1, N, B).astype(np.int64)), \
        t(rs.randint(0, N, B).astype(np.int64))
    loss, _, _, dWu, dWi, dbu, dbi = ops.mf_bloom_train_step(*base, users, items, negs, 0, 1, [], SEEDS[:H], -1, 0, False)
    lr = 0.01 / float(max(dWu.abs().max(), dWi.abs().max()))
    p1 = [x.clone() for x in base]
    l1 = ops.mf_bloom_train_step_inplace(*p1, users, items, negs, 'pointwise', 1, [], SEEDS[:H], -1, 0, _lib.OPT_SGD, lr)
    assert_close(l1.item(), loss.item(), 1e-6, what='loss')
    for p, b0, gr, nm in zip(p1, base, (dWu, dWi, dbu, dbi), ('Wu', 'Wi', 'bu', 'bi')):
        assert_close_dev(p, b0 - lr * gr.reshape(b0.shape), 2e-6, what=nm)
    p2 = [x.clone() for x in base]
    st = [torch.zeros_like(x) for x in p2]
    ops.mf_bloom_train_step_inplace(*p2, users, items, negs, 'pointwise', 1, [], SEEDS[:H], -1, 0, _lib.OPT_ADAGRAD,
                                    0.05, states=st)
    for s_, gr, nm in zip(st, (dWu, dWi, dbu, dbi), ('sWu', 'sWi', 'sbu', 'sbi')):
        assert_close_dev(s_, (gr * gr).reshape(s_.shape), 2e-5, atol=1e-30, what=nm)
    p3 = [x.clone() for x in base]
    st3 = [torch.zeros_like(x) for x in p3]
    ops.mf_bloom_train_step_inplace(*p3, users, items, negs, 'pointwise', 1, [], SEEDS[:H], -1, 0, _lib.OPT_ADAGRAD,
                                    0.05, states=st3)
    for x, y in zip(p2 + st, p3 + st3):
        assert torch.equal(x, y), 'fused hashed step is not bit-reproducible'


def test_fused_bloom_both_sides_vs_generic_route():
    """Bloom on users *and* items (the reference's own MF Bloom test shape,
    tests/factorization/test_implicit.py:127-164): fused step == generic autograd route."""
    from spotlight_b200 import losses, ops
    from spotlight_b200.factorization.representations import BilinearNet
    from spotlight_b200.layers import BloomEmbedding
    torch.manual_seed(0)
    U, I, D, B = 300, 500, 32, 512
    net = BilinearNet(U, I, D, user_embedding_layer=BloomEmbedding(U, D, compression_ratio=0.5,
                                                                    num_hash_functions=2),
                      item_embedding_layer=BloomEmbedding(I, D, compression_ratio=0.4,
                                                          num_hash_functions=3)).to(dev())
    with torch.no_grad():
        net.user_biases.weight.normal_(0, 0.1)
        net.item_biases.weight.normal_(0, 0.1)
    rs = np.random.RandomState(3)
    users, items, negs = (t(rs.randint(0, n, B).astype(np.int64)) for n in (U, I, I))
    spec = net.fused_spec()
    assert spec is not None and len(spec['user_seeds']) == 2 and len(spec['item_seeds']) == 3
    lf = ops.fused_bloom_loss(spec['Wu'], spec['Wi'], net.user_biases.weight, net.item_biases.weight,
                              users, items, negs, 'pointwise', 1, spec)
    lf.backward()
    got = {k: p.grad.clone() for k, p in net.named_parameters()}
    net.zero_grad()
    lg = losses.pointwise_loss(net(users, items), net(users, negs))
    lg.backward()
    assert_close(lf.item(), lg.item(), 1e-5, what='loss')
    for k, p in net.named_parameters():
        assert_close(got[k].cpu().numpy(), p.grad.cpu().numpy(), 1e-5, atol=1e-8, what=k)


def test_model_routes_bloom_through_fused_step():
    from spotlight_b200.factorization.implicit import ImplicitFactorizationModel
    from spotlight_b200.factorization.representations import BilinearNet
    from spotlight_b200.interactions import Interactions
    from spotlight_b200.layers import BloomEmbedding, ScaledEmbedding
    rs = np.random.RandomState(0)
    inter = Interactions(rs.randint(0, 100, 2000).astype(np.int32), rs.randint(0, 400, 2000).astype(np.int32),
                         num_users=100, num_items=400)
    rep = BilinearNet(100, 400, 16, user_embedding_layer=ScaledEmbedding(100, 16),
                      item_embedding_layer=BloomEmbedding(400, 16, compression_ratio=0.5, num_hash_functions=2))
    model = ImplicitFactorizationModel(loss='bpr', embedding_dim=16, batch_size=256, n_iter=2,
                                       representation=rep, use_cuda=True,
                                       random_state=np.random.RandomState(1))
    model.fit(inter)
    assert model._route() == 'bloom'
    assert model.predict(3).shape == (400,)


# ------------------------------------------------------------------- losses

@pytest.mark.parametrize('kind', ['pointwise', 'bpr', 'hinge', 'adaptive_hinge'])
@pytest.mark.parametrize('masked', [False, True])
def test_loss_ops_vs_oracle(kind, masked):
    from spotlight_b200 import losses
    rs = np.random.RandomState(2)
    shape = (37, 11)
    pos = rs.randn(*shape).astype(np.float32)
    neg = rs.randn(*((4,) + shape if kind == 'adaptive_hinge' else shape)).astype(np.float32)
    mask = (rs.rand(*shape) > 0.3) if masked else None
    lref, gp, gn = omf.loss_and_score_grads(kind, pos, neg, mask, np.float64)
    p, n = t(pos).requires_grad_(), t(neg).requires_grad_()
    fn = getattr(losses, kind + '_loss')
    l = fn(p, n, mask=t(mask) if masked else None)
    l.backward()
    assert_close(l.item(), lref, 1e-5, what='loss')
    assert_close(p.grad.cpu().numpy(), gp, 1e-5, what='gpos')
    assert_close(n.grad.cpu().numpy(), gn, 1e-5, what='gneg')
