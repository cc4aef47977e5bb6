"""Per-launch device times of one forward (CUDA events around every launch of the profiled
classes): writes layers_b{clips}_{size}.csv into the directory given as the third argument (default: a temporary
directory) and prints the GEMM layers sorted by time."""
import collections
import csv
import os
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from archs.pgtformer_arch import PGTFormer  # noqa: E402
from pgtformer_b200 import ops  # noqa: E402

clips = int(sys.argv[1]) if len(sys.argv) > 1 else 16
size = int(sys.argv[2]) if len(sys.argv) > 2 else 512
kw = dict(bench.load_network_g())
kw.pop('type')
m = PGTFormer(**kw).cuda()
m.eval()
x = torch.rand(clips * 3, 3, size, size).cuda()
for _ in range(2):
    m(x, w=1, adain=True)
torch.cuda.synchronize()
out_dir = sys.argv[3] if len(sys.argv) > 3 else tempfile.mkdtemp(prefix='pgt_layers_')
os.makedirs(out_dir, exist_ok=True)
path = os.path.join(out_dir, 'layers_b%d_%d.csv' % (clips, size))
ops.profile_begin()
m(x, w=1, adain=True)
prof = ops.profile_end(path)
print({k: (round(v[1], 3), v[2]) for k, v in prof.items() if v[2]})
agg = collections.OrderedDict()
for r in csv.DictReader(open(path)):
    if r['class'] != '0':
        continue
    a = agg.setdefault(r['desc'], [0, 0.0, 0.0])
    a[0] += 1
    a[1] += float(r['ms'])
    a[2] += float(r['work'])
tot = sum(a[1] for a in agg.values())
print('gemm total ms %.2f' % tot)
for d, a in sorted(agg.items(), key=lambda kv: -kv[1][1]):
    print('%-58s n=%2d %8.3f ms %5.1f%% %7.1f TF/s' % (d, a[0], a[1], 100 * a[1] / tot, a[2] / a[1] / 1e9))
