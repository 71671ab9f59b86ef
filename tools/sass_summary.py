"""SASS evidence for the wgmma / TMA kernels: per-kernel counts of the Hopper tensor-core, TMA and mbarrier mnemonics in the
built .so (`cuobjdump -sass`), plus a short excerpt around the first HGMMA of each kernel.  CPU-only (no GPU needed).

    python tools/sass_summary.py > sass_summary.md
"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, 'novel_view_synthesis_3d_b200', 'libxunet_b200.so')
MNEMONICS = ['HGMMA', 'WARPGROUP', 'UTMALDG', 'UTMASTG', 'UTMAREDG', 'UTMAPF', 'UBLKCP', 'SYNCS', 'REDG', 'RED.E', 'ATOMG', 'DADD', 'HMMA', 'MUFU.EX2', 'SHFL']


def main():
    sass = subprocess.run(['cuobjdump', '-sass', LIB], capture_output=True, text=True, check=True).stdout
    kernels, cur = collections.OrderedDict(), None
    for line in sass.splitlines():
        m = re.search(r'Function : (\S+)', line)
        if m:
            cur = m.group(1)
            kernels[cur] = []
        elif cur is not None:
            kernels[cur].append(line)
    demangle = lambda n: subprocess.run(['c++filt', n], capture_output=True, text=True).stdout.strip()
    print('# SASS summary of libxunet_b200.so (cuobjdump -sass, sm_90a)\n')
    print('Counts of Hopper-native mnemonics per kernel (wgmma.mma_async -> HGMMA, wgmma fence / commit / wait -> WARPGROUP, '
          'TMA -> UTMALDG/UTMASTG/UTMAREDG/UBLKCP, mbarrier -> SYNCS, fp64 reductions -> DADD / RED.E).  HMMA = legacy mma.sync.\n')
    print('| kernel | instr | ' + ' | '.join(MNEMONICS) + ' |')
    print('|---|---|' + '---|' * len(MNEMONICS))
    total = collections.Counter()
    excerpts = []
    for name, lines in kernels.items():
        ins = [l for l in lines if re.search(r'/\*[0-9a-f]{4}\*/', l)]
        cnt = {mn: sum(1 for l in ins if re.search(r'(?<![A-Z])' + re.escape(mn), l)) for mn in MNEMONICS}
        if not any(cnt[mn] for mn in ('HGMMA', 'UTMALDG', 'UBLKCP')):
            continue
        total.update(cnt)
        short = re.sub(r'\(.*', '', demangle(name).replace('(anonymous namespace)::', '')).replace('void ', '')
        print(f'| `{short}` | {len(ins)} | ' + ' | '.join(str(cnt[mn]) for mn in MNEMONICS) + ' |')
        for i, l in enumerate(ins):
            if 'HGMMA' in l:
                excerpts.append((short, [re.sub(r'\s+', ' ', x.strip()) for x in ins[max(0, i - 3):i + 4]]))
                break
    print('| **total** | | ' + ' | '.join(str(total[mn]) for mn in MNEMONICS) + ' |\n')
    print('## Excerpts (first tensor-core instruction of each kernel, +-3 instructions)\n')
    for short, ex in excerpts[:12]:
        print(f'`{short}`\n```')
        print('\n'.join(ex))
        print('```')


if __name__ == '__main__':
    main()
