"""Host against device data preparation: Interactions.to_sequence (L = 200, step = L; and
L = 50, step = 1) and both train/test splits, over n interactions of 1M users.

Usage: python profiles/bench_prepare.py [--n 100000000] [--reps 3]

Each workload first checks that the device outputs equal the host outputs, then reports the
host time (one run) and the device time (median of --reps runs after one warm-up), each on a
host clock that ends in a device synchronise.  The L = 50, step = 1 workload writes n rows of
50, so it runs at n / 10 to keep the host arrays in memory.  Prints the card name and power
limit with the numbers.
"""

import argparse
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from spotlight_b200.cross_validation import random_train_test_split, user_based_train_test_split  # noqa: E402
from spotlight_b200.interactions import Interactions  # noqa: E402

COLUMNS = ('user_ids', 'item_ids', 'ratings', 'timestamps', 'weights')


def card():
    out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                         capture_output=True, text=True)
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 else torch.cuda.get_device_name(0)


def data(n, seed=0):
    rs = np.random.RandomState(seed)
    return Interactions(rs.randint(0, 10 ** 6, n).astype(np.int32), rs.randint(1, 10 ** 5, n).astype(np.int32),
                        timestamps=rs.randint(0, 10 ** 9, n).astype(np.int64), num_users=10 ** 6, num_items=10 ** 5)


def to_device(inter):
    kw = {k: None if getattr(inter, k) is None else torch.from_numpy(getattr(inter, k)).cuda() for k in COLUMNS}
    return Interactions(kw.pop('user_ids'), kw.pop('item_ids'), num_users=inter.num_users,
                        num_items=inter.num_items, **kw)


def timed(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, time.perf_counter() - t


def same(a, b):
    if torch.is_tensor(b):
        return np.array_equal(a, b.cpu().numpy())
    return all(same(getattr(a, k), getattr(b, k)) for k in COLUMNS if getattr(a, k) is not None)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--n', type=int, default=10 ** 8)
    ap.add_argument('--reps', type=int, default=3)
    args = ap.parse_args()
    print('card: %s' % card())
    workloads = [
        ('to_sequence L=200 step=200', args.n, lambda d: d.to_sequence(200),
         lambda s: (s.sequences, s.user_ids)),
        ('to_sequence L=50 step=1', args.n // 10, lambda d: d.to_sequence(50, step_size=1),
         lambda s: (s.sequences, s.user_ids)),
        ('random_train_test_split', args.n,
         lambda d: random_train_test_split(d, random_state=np.random.RandomState(1)), lambda s: s),
        ('user_based_train_test_split', args.n,
         lambda d: user_based_train_test_split(d, random_state=np.random.RandomState(1)), lambda s: s),
    ]
    cache = {}
    for name, n, fn, parts in workloads:
        if n not in cache:
            cache.clear()
            host = data(n)
            cache[n] = (host, to_device(host))
        host, dev = cache[n]
        h_out, h_time = timed(lambda: fn(host))
        d_out, _ = timed(lambda: fn(dev))
        ok = all(same(a, b) for a, b in zip(parts(h_out), parts(d_out)))
        del h_out, d_out
        if not ok:
            raise SystemExit('%s: device output differs from the host output' % name)
        times = []
        for _ in range(args.reps):
            out, t = timed(lambda: fn(dev))
            del out
            times.append(t)
        d_time = float(np.median(times))
        print('%-28s n=%-10d host %8.3f s  device %8.4f s  (%.0fx)' % (name, n, h_time, d_time, h_time / d_time))


if __name__ == '__main__':
    main()
