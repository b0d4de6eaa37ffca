"""GPU tests of the shard kernels on one device, no process group: the owner bucketing of the row
exchange (slb_unique_bucket, through GpuBackend.unique_bucket) against NumpyBackend.unique_bucket,
the member gather of the dense-exchange epoch (slb_shard_gather_batch) against NumPy fancy
indexing, and the owner-shard Adagrad (slb_adagrad_dense) against NumpyBackend.adagrad_dense --
at row spaces of one, several and hundreds of 4096-row scan tiles, up to eight owners, and
grid-stride lengths past one pass."""

import os
import sys

import numpy as np
import pytest
import torch

from conftest import ROOT

sys.path.insert(0, os.path.join(ROOT, 'tests'))
pytestmark = pytest.mark.gpu

import sharded_common as sc            # noqa: E402

DEV = torch.device('cuda', 0)
TILE = 4096                            # segindex.cuh's scan tile


def _lib():
    from spotlight_b200 import _lib
    return _lib.load()


def _dev(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


# ------------------------------------------------------------------ owner bucketing

ROWS = [1, TILE - 1, TILE, TILE + 1, 3 * TILE + 17, 100000, 1000003]
PATTERNS = ['uniform', 'equal', 'end_owners', 'permutation', 'edges']


def _sizes(rows):
    return sorted({1, 37, max(1, rows // 3), min(4 * rows, (1 << 22) + 5)})


def _owners(rows):
    """(chunk, nparts): ceil(rows / nparts) for 1, 2, 3 and 8 owners, and 8 owners on a chunk
    sized for 5, so the last owners' ranges are empty or lie wholly past the row space."""
    return [(-(-rows // p), p) for p in (1, 2, 3, 8)] + [(-(-rows // 5), 8)]


def _ids(pattern, rows, n, chunk, nparts, rs):
    if pattern == 'uniform':
        return rs.randint(0, rows, n)
    if pattern == 'equal':
        return np.full(n, rs.randint(0, rows))
    if pattern == 'end_owners':
        # owner 0 and the last owner with rows: every owner between them gets none
        last = min(nparts - 1, (rows - 1) // chunk)
        lo0, hi0 = 0, min(chunk, rows)
        lo1, hi1 = last * chunk, min((last + 1) * chunk, rows)
        pick = rs.randint(0, 2, n).astype(bool)
        return np.where(pick, rs.randint(lo0, hi0, n), rs.randint(lo1, hi1, n))
    if pattern == 'permutation':
        return rs.permutation(rows)
    edges = np.array([r for r in (0, rows - 1, TILE - 1, TILE) if r < rows])
    return edges[rs.randint(0, len(edges), n)]


def _bucket(be, ids, rows, chunk, nparts):
    uniq, inverse, bounds = be.unique_bucket(_dev(ids.astype(np.int64)), rows, chunk, nparts)
    return uniq.cpu().numpy(), inverse.cpu().numpy(), bounds


def _check_bucket(got, ids, rows, chunk, nparts, what):
    want_u, want_inv, want_b = sc.NumpyBackend().unique_bucket(torch.from_numpy(ids.astype(np.int64)), rows,
                                                               chunk, nparts)
    uniq, inverse, bounds = got
    assert np.array_equal(uniq, want_u.numpy()), what + ': uniq'
    assert np.array_equal(inverse, want_inv.numpy()), what + ': inverse'
    assert bounds == want_b, (what + ': owner boundaries', bounds, want_b)
    assert bounds[-1] == len(uniq), what + ': total'


@pytest.mark.parametrize('rows', ROWS)
def test_unique_bucket_matches_numpy(rows):
    """Distinct ids ascending, the inverse map, the nparts + 1 owner boundaries and the total are
    NumpyBackend.unique_bucket's exactly, for sparse requests, heavy duplication, one id, every row
    once, ids on the row space's and the scan tile's edges, and owners that get no ids between
    owners that do; two runs on the cached workspace are bit-identical."""
    from spotlight_b200.sharded import GpuBackend
    be = GpuBackend(DEV)
    rs = np.random.RandomState(rows % 1000)
    for pattern in PATTERNS:
        for n in (_sizes(rows) if pattern != 'permutation' else [rows]):
            for chunk, nparts in _owners(rows):
                ids = _ids(pattern, rows, n, chunk, nparts, rs)
                what = '%s n=%d chunk=%d nparts=%d' % (pattern, len(ids), chunk, nparts)
                got = _bucket(be, ids, rows, chunk, nparts)
                _check_bucket(got, ids, rows, chunk, nparts, what)
                if pattern == 'uniform' and nparts == 8:
                    again = _bucket(be, ids, rows, chunk, nparts)
                    assert all(np.array_equal(a, b) for a, b in zip(got[:2], again[:2])) and got[2] == again[2], what


@pytest.mark.parametrize('rows', [3 * TILE + 17, 1000003])
def test_unique_bucket_workspace_reuse(rows):
    """The workspace's counters are zero at rest: a call repeated on the cached workspace, and
    repeated after a call with another n (which sizes the workspace differently), gives the same
    result bit for bit."""
    from spotlight_b200.sharded import GpuBackend
    be = GpuBackend(DEV)
    rs = np.random.RandomState(3)
    chunk, nparts = -(-rows // 3), 3
    a = rs.randint(0, rows, rows // 3)
    b = rs.randint(0, rows, min(4 * rows, 1 << 22))
    first = _bucket(be, a, rows, chunk, nparts)
    _check_bucket(first, a, rows, chunk, nparts, 'first')
    second = _bucket(be, a, rows, chunk, nparts)
    _check_bucket(_bucket(be, b, rows, chunk, nparts), b, rows, chunk, nparts, 'other n')
    third = _bucket(be, a, rows, chunk, nparts)
    for got in (second, third):
        assert all(np.array_equal(x, y) for x, y in zip(first[:2], got[:2])) and first[2] == got[2]


@pytest.mark.parametrize('bad', ['negative', 'rows'])
def test_unique_bucket_rejects_out_of_range_ids(bad):
    """An id outside [0, rows) raises ValueError instead of being trained as row 0, and the next
    valid call on the same cached workspace succeeds with the right result."""
    from spotlight_b200.sharded import GpuBackend
    be = GpuBackend(DEV)
    rows, chunk, nparts = 3 * TILE + 17, TILE + 6, 3
    rs = np.random.RandomState(5)
    ids = rs.randint(0, rows, 5000)
    _check_bucket(_bucket(be, ids, rows, chunk, nparts), ids, rows, chunk, nparts, 'before')
    bad_ids = ids.copy()
    bad_ids[1234] = -1 if bad == 'negative' else rows
    with pytest.raises(ValueError):
        _bucket(be, bad_ids, rows, chunk, nparts)
    _check_bucket(_bucket(be, ids, rows, chunk, nparts), ids, rows, chunk, nparts, 'after')


def test_unique_bucket_rejections():
    """Null pointers, n <= 0, bad sizes, chunk * nparts < rows and a short workspace are rejected
    with an error code before any launch: the outputs keep their contents."""
    from spotlight_b200 import ops
    lib = _lib()
    rows, n, nparts = 1000, 300, 4
    chunk = -(-rows // nparts)
    ids = _dev(np.random.RandomState(1).randint(0, rows, n).astype(np.int64))
    uniq = torch.full((n,), -7, dtype=torch.int64, device=DEV)
    inverse = torch.full((n,), -7, dtype=torch.int64, device=DEV)
    counts = torch.full((nparts + 2,), -7, dtype=torch.int64, device=DEV)
    need = lib.slb_unique_workspace_bytes(n, rows)
    ws = torch.zeros(need, dtype=torch.uint8, device=DEV)
    P = ops._ptr

    def call(ids_p=P(ids), nn=n, nrows=rows, ch=chunk, parts=nparts, u=P(uniq), inv=P(inverse), c=P(counts),
             wsp=P(ws), wsb=need):
        return lib.slb_unique_bucket(ids_p, nn, nrows, ch, parts, u, inv, c, wsp, wsb, ops._stream())

    for bad in (dict(ids_p=None), dict(u=None), dict(inv=None), dict(c=None), dict(wsp=None), dict(nn=0),
                dict(nn=-1), dict(nrows=0), dict(ch=0), dict(parts=0), dict(ch=chunk - 1), dict(parts=nparts - 1),
                dict(wsb=need - 1)):
        assert call(**bad) != 0, bad
        assert lib.slb_last_error()
    torch.cuda.synchronize()
    for t in (uniq, inverse, counts):
        assert (t == -7).all()
    assert call() == 0
    torch.cuda.synchronize()
    assert int(counts[nparts]) == int(counts[nparts + 1]) == len(np.unique(ids.cpu().numpy()))


# ------------------------------------------------------------------ member gather


@pytest.mark.parametrize('n_neg', [1, 2, 5])
@pytest.mark.parametrize('m', [0, 1, 1000, 600000])
def test_shard_gather_batch_matches_numpy(m, n_neg):
    """users_out = users[pos] - user_lo, items_out = items[pos], negs_out = the n_neg negatives of
    each member from a negatives array that holds only the slice from neg_base on; m = 0 leaves
    the outputs untouched; 600000 members take more than one grid-stride pass."""
    from spotlight_b200 import ops
    lib = _lib()
    rs = np.random.RandomState(m + n_neg)
    N, neg_base, span, user_lo = 2000000, 700001, 900000, 123457
    users = rs.randint(user_lo, user_lo + 1000000, N).astype(np.int64)
    items = rs.randint(0, 100000, N).astype(np.int64)
    pos = np.sort(rs.choice(span, size=m, replace=False)).astype(np.int64) + neg_base
    # the negatives of positions neg_base .. neg_base + span; the allocation runs on past the slice
    # (as a chunk of a longer stream does), so that a gather which ignored neg_base reads wrong
    # values rather than unallocated memory
    negs_mem = rs.randint(0, 100000, (neg_base + span + neg_base) * n_neg).astype(np.int64)
    negs = negs_mem[:span * n_neg]
    cap = max(m, 1)
    outs = [torch.full((k,), -7, dtype=torch.int64, device=DEV) for k in (cap, cap, cap * n_neg)]
    d_pos, d_u, d_i, d_n = (_dev(x) for x in (pos, users, items, negs_mem))
    P = ops._ptr
    rc = lib.slb_shard_gather_batch(P(d_pos), m, P(d_u), P(d_i), P(d_n), neg_base, n_neg, user_lo,
                                    P(outs[0]), P(outs[1]), P(outs[2]), ops._stream())
    assert rc == 0
    torch.cuda.synchronize()
    got = [o.cpu().numpy() for o in outs]
    if m == 0:
        assert all((g == -7).all() for g in got)
        return
    assert np.array_equal(got[0], users[pos] - user_lo)
    assert np.array_equal(got[1], items[pos])
    want = negs.reshape(span, n_neg)[pos - neg_base].reshape(-1)
    assert np.array_equal(got[2], want)


def test_shard_gather_batch_rejections():
    """Null pointers and n_neg < 1 are rejected before any launch when there are members."""
    from spotlight_b200 import ops
    lib = _lib()
    x = torch.zeros(8, dtype=torch.int64, device=DEV)
    out = torch.full((8,), -7, dtype=torch.int64, device=DEV)
    P = ops._ptr
    args = [P(x), 4, P(x), P(x), P(x), 0, 1, 0, P(out), P(out), P(out)]
    for k in (0, 2, 3, 4, 8, 9, 10):
        bad = list(args)
        bad[k] = None
        assert lib.slb_shard_gather_batch(*bad, ops._stream()) != 0, k
        assert lib.slb_last_error()
    bad = list(args)
    bad[6] = 0
    assert lib.slb_shard_gather_batch(*bad, ops._stream()) != 0
    torch.cuda.synchronize()
    assert (out == -7).all()


# ------------------------------------------------------------------ owner-shard Adagrad


def _adagrad_case(n, state, seed):
    rs = np.random.RandomState(seed)
    W = rs.randn(n).astype(np.float32)
    S = np.zeros(n, np.float32) if state == 'zero' else (np.abs(rs.randn(n)) * 1e-2).astype(np.float32)
    scale = rs.choice(np.array([1e-8, 1e-3, 1.0, 1e3]), n)              # tiny to large gradients
    G = (rs.randn(n) * scale).astype(np.float32)
    G[rs.rand(n) < 0.3] = 0.0                                          # about 30 % exact zeros
    if n >= 3:
        G[0], G[1] = 0.0, 1e3
    return W, S, G


@pytest.mark.parametrize('state', ['zero', 'positive'])
@pytest.mark.parametrize('n', [1, 3, 1000, 2000003])
def test_adagrad_dense_matches_numpy(n, state):
    """torch.optim.Adagrad's update (lr_decay 0) elementwise against NumpyBackend.adagrad_dense in
    float64: elements with a zero gradient keep W and the accumulator bit for bit; the others are
    within a few float32 ulps of max(|W|, |dW|) (IEEE sqrtf and division, the same expression);
    2000003 elements take more than one grid-stride pass."""
    from spotlight_b200.sharded import GpuBackend
    lr, eps = 0.05, 1e-10
    W, S, G = _adagrad_case(n, state, n)
    dW, dS = _dev(W), _dev(S)
    GpuBackend(DEV).adagrad_dense(dW, dS, _dev(G), lr, eps)
    torch.cuda.synchronize()
    gw, gs = dW.cpu().numpy().astype(np.float64), dS.cpu().numpy().astype(np.float64)
    rw, rs_ = torch.from_numpy(W.copy()), torch.from_numpy(S.copy())
    sc.NumpyBackend().adagrad_dense(rw, rs_, torch.from_numpy(G), lr, eps)    # float64, rounded once
    rw, rs_ = rw.numpy().astype(np.float64), rs_.numpy().astype(np.float64)
    zero = G == 0
    assert np.array_equal(gw[zero], W[zero]) and np.array_equal(gs[zero], S[zero])
    nz = ~zero
    ulp_w = np.spacing(np.maximum(np.abs(W), np.abs(rw - W)).astype(np.float32)).astype(np.float64)
    ulp_s = np.spacing(rs_.astype(np.float32)).astype(np.float64)
    assert (np.abs(gw - rw)[nz] <= 4 * ulp_w[nz]).all(), np.abs(gw - rw)[nz].max()
    assert (np.abs(gs - rs_)[nz] <= 2 * ulp_s[nz]).all(), np.abs(gs - rs_)[nz].max()
    assert (gw[nz] != W[nz]).any() or n < 3


def test_adagrad_dense_empty_and_rejections():
    """n <= 0 is a no-op that needs no storage; null pointers are rejected before any launch."""
    from spotlight_b200 import ops
    lib = _lib()
    W = torch.ones(16, device=DEV)
    S = torch.ones(16, device=DEV)
    G = torch.ones(16, device=DEV)
    P = ops._ptr
    assert lib.slb_adagrad_dense(None, None, None, 0, 0.05, 1e-10, ops._stream()) == 0
    assert lib.slb_adagrad_dense(P(W), P(S), P(G), -1, 0.05, 1e-10, ops._stream()) == 0
    for bad in ((None, P(S), P(G)), (P(W), None, P(G)), (P(W), P(S), None)):
        assert lib.slb_adagrad_dense(*bad, 16, 0.05, 1e-10, ops._stream()) != 0
        assert lib.slb_last_error()
    torch.cuda.synchronize()
    assert (W == 1).all() and (S == 1).all()
