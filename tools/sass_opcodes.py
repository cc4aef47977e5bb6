#!/usr/bin/env python
"""Per-kernel SASS opcode census of libpgt_b200.so (cuobjdump -sass): which instructions each kernel really runs on
sm_90a.  HGMMA = wgmma, UTMALDG / UTMASTG / UTMAPF = TMA loads / stores / prefetches, SYNCS = mbarrier operations,
HMMA = warp-level mma.sync.
    python tools/sass_opcodes.py
"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, 'pgtformer_b200', 'lib', 'libpgt_b200.so')
OPS = ['HGMMA', 'UTMALDG', 'UTMASTG', 'UTMAPF', 'UBLKCP', 'SYNCS', 'HMMA', 'LDGSTS', 'MUFU', 'DFMA', 'FFMA']


def main():
    out = subprocess.run(['cuobjdump', '-sass', LIB], stdout=subprocess.PIPE, text=True, check=True).stdout
    counts = collections.OrderedDict()
    cur = None
    for line in out.splitlines():
        m = re.search(r'Function : (\S+)', line)
        if m:
            name = subprocess.run(['c++filt', m.group(1)], stdout=subprocess.PIPE, text=True).stdout.strip()
            name = re.sub(r'\(.*', '', name)
            cur = counts.setdefault(name, collections.Counter())
            continue
        if cur is None:
            continue
        m = re.match(r'\s+/\*[0-9a-f]+\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)', line)
        if m:
            op = m.group(1)
            for o in OPS:
                if op.startswith(o):
                    cur[o] += 1
    print('# SASS opcode counts per kernel of %s (cuobjdump -sass, sm_90a)' % os.path.relpath(LIB, ROOT))
    print('%-58s' % 'kernel' + ''.join('%9s' % o for o in OPS))
    for k, c in counts.items():
        print('%-58s' % k[:57] + ''.join('%9d' % c[o] for o in OPS))


if __name__ == '__main__':
    main()
