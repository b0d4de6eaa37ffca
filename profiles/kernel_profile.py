"""Per-kernel durations of the bench.py epoch (BPR MF, 1M x 100K x 64, B = 524288, fused Adagrad)
under torch.profiler, in a run of its own.

    python profiles/kernel_profile.py [--steps K] [--warmup W] [--out DIR]

Times the same epoch twice: with the plan on its own stream (what fit() does) and with
SLB_PLAN_SAME_STREAM=1 (plan serialised in front of the float kernels), so the cost of the plan
under overlap can be read off.  Prints one JSON line: the card name and power limit, and for each
mode the average duration and launch count of every kernel in the epoch and the epoch's wall time
per step.  The kernel traces are written under DIR when --out is given."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def card():
    import torch
    out = {'name': torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        out['power_limit'], out['max_sm_clock'] = [x.strip() for x in q[0].split(',')]
    except Exception as exc:            # the line says so instead of inventing a limit
        out['power_limit'] = 'unknown (%s)' % repr(exc)[:80]
    return out


def profile_epoch(a, same_stream, out_dir):
    import torch
    from torch.profiler import profile, ProfilerActivity
    from bench import build_model
    if same_stream:
        os.environ['SLB_PLAN_SAME_STREAM'] = '1'
    else:
        os.environ.pop('SLB_PLAN_SAME_STREAM', None)
    model = build_model(a, 0)
    dev = torch.device('cuda', 0)
    B, K, W = a.batch, a.steps, a.warmup
    g = torch.Generator(device=dev).manual_seed(1234)
    users = torch.randint(0, a.users, ((K + W) * B,), device=dev, generator=g)
    items = torch.randint(0, a.items, ((K + W) * B,), device=dev, generator=g)
    model._run_epoch_device(users[:W * B], items[:W * B])
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        model._run_epoch_device(users[W * B:], items[W * B:])
        e1.record()
        torch.cuda.synchronize()
    kernels = {}
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        k = kernels.setdefault(e.name, [0, 0.0])
        k[0] += 1
        k[1] += e.device_time_total if hasattr(e, 'device_time_total') else e.cuda_time_total
    if out_dir:
        os.makedirs(out_dir, exist_ok=True)
        prof.export_chrome_trace(os.path.join(out_dir, 'epoch_%s.pt.trace.json'
                                              % ('same_stream' if same_stream else 'two_streams')))
    table = {n: {'calls': c, 'avg_ms': t / c / 1e3} for n, (c, t) in kernels.items()}
    table = dict(sorted(table.items(), key=lambda kv: -kv[1]['avg_ms'] * kv[1]['calls']))
    del model, users, items
    torch.cuda.empty_cache()
    return {'ms_per_step_profiled': e0.elapsed_time(e1) / K, 'kernels': table}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=50)
    ap.add_argument('--warmup', type=int, default=10)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    a = argparse.Namespace(batch=524288, users=1_000_000, items=100_000, dim=64, loss='bpr', lr=0.05,
                           steps=args.steps, warmup=args.warmup)
    line = {'card': card(), 'config': 'BPR MF 1M x 100K x 64, B = 524288, fused Adagrad, %d steps' % a.steps,
            'two_streams': profile_epoch(a, False, args.out),
            'same_stream': profile_epoch(a, True, args.out)}
    print(json.dumps(line))


if __name__ == '__main__':
    np.seterr(all='ignore')
    main()
