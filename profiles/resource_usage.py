"""Per-kernel registers / stack / static shared memory / local memory of the built library.

    python profiles/resource_usage.py > profiles/resource_usage_rNN.txt

Reads `cuobjdump --dump-resource-usage spotlight_b200/libspotlight_b200.so` (no GPU needed).
LOCAL > 0 or STACK > 0 on a hot kernel means spills: check before spending GPU time."""
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
so = os.path.join(ROOT, 'spotlight_b200', 'libspotlight_b200.so')
txt = subprocess.run(['cuobjdump', '--dump-resource-usage', so], capture_output=True, text=True).stdout
rows, cur = [], None
for line in txt.splitlines():
    m = re.match(r'\s*Function (\S+):', line)
    if m:
        cur = m.group(1)
        continue
    m = re.match(r'\s*REG:(\d+) STACK:(\d+) SHARED:(\d+) LOCAL:(\d+)', line)
    if m and cur:
        rows.append((cur,) + tuple(int(x) for x in m.groups()))
        cur = None
names = subprocess.run(['c++filt'], input='\n'.join(r[0] for r in rows), capture_output=True,
                       text=True).stdout.splitlines()
print('# cuobjdump --dump-resource-usage spotlight_b200/libspotlight_b200.so  (sm_90a, -O3 -lineinfo)')
print('# %d kernels; regs  stack  static_smem  local  kernel' % len(rows))
out = []
for (n, reg, stack, sh, loc), d in zip(rows, names):
    d = re.sub(r'\(anonymous namespace\)::', '', d)
    d = re.sub(r'^void ', '', d)
    d = re.sub(r'\((?:[^()]|\([^()]*\))*\)$', '', d)
    out.append((d, reg, stack, sh, loc))
for d, reg, stack, sh, loc in sorted(out):
    print('%5d %6d %12d %6d  %s' % (reg, stack, sh, loc, d[:140]))

# Dynamic shared memory of the LSTM recurrence kernels per CTA: csrc/seq.cu lstm_cluster_size /
# lstm_dev and csrc/seq_lstm.cuh fwd_smem_floats / bwd_smem_floats restated.
print('# lstm_fwd_kernel / lstm_bwd_kernel dynamic shared memory per CTA')
print('#   D  cluster  units  seqs/tile   fwd_bytes   bwd_bytes')
for D in (4, 32, 64, 100, 128, 132, 256):
    c = 1 if D <= 64 else (4 if D <= 128 else 8)
    U = -(-D // c)
    NB = min(max(256 // U, 1), 32)
    fwd = 4 * U * D + 4 * U + 2 * NB * (D + 4)
    bwd = 4 * U * D + 4 * NB * U + 2 * NB * D
    print('%5d %8d %6d %10d %11d %11d' % (D, c, U, NB, 4 * fwd, 4 * bwd))
