#!/usr/bin/env python
"""Opcode histogram per kernel from the built objects (cuobjdump -sass): the evidence that the hot loops are what DESIGN.md says they are
(128-bit streaming loads / stores, shared-memory atomics with hardware aggregation, no IEEE-division expansion in the loop, TMA bulk copies
only in the TMA variant, no tensor-core instructions anywhere -- nothing on this path is a contraction).

    python tools/sass_summary.py > profiles/r02_sass_opcodes.md
"""
import collections
import glob
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KEYS = ['LDG.E.128', 'LDG.E.NA.128', 'LDG.E', 'STG.E.128', 'STG.E', 'LDS', 'STS', 'ATOMS', 'ATOMG', 'RED', 'REDUX', 'SHFL', 'BAR', 'MUFU.RCP', 'FCHK', 'F2I',
        'FFMA', 'FMUL', 'IMAD', 'UBLKCP', 'SYNCS', 'UTCHMMA', 'UTCQMMA', 'HMMA', 'DADD', 'DMUL', 'DFMA', 'MUFU.LG2', 'CALL']


def demangle(names):
    out = subprocess.run(['c++filt'], input='\n'.join(names), capture_output=True, text=True).stdout.split('\n')
    return dict(zip(names, out))


def short(name):
    name = re.sub(r'ppqb::', '', name)
    name = re.sub(r'\(.*$', '', name)
    name = name.replace('void ', '')
    return name if len(name) <= 110 else name[:107] + '...'


def main():
    objs = sorted(glob.glob(os.path.join(ROOT, 'ppq_b200', '_build', '*.o')))
    wanted = sys.argv[1:]                                               # optional substrings to filter kernel names
    print('# SASS opcode histogram per kernel (sm_90a, cuobjdump -sass of ppq_b200/_build/*.o)\n')
    print('Columns: total instructions, then the opcodes that characterise the kernel. `LDG.128` counts every 128-bit global load '
          '(`LDG.E.128*`, incl. the `.NA` no-allocate / `.CONSTANT` forms), `ATOMS` the shared-memory atomics (`ATOMS.POPC.INC` = hardware-aggregated '
          'increment), `RED/ATOMG` global reductions, `RCP/FCHK` the reciprocal and the IEEE-division range check (FCHK only appears in the '
          'out-of-line slow path), `UBLKCP/SYNCS` TMA bulk copies and mbarrier operations, `MMA` any tensor-core instruction.\n')
    for obj in objs:
        if not obj.endswith('.o') or 'host' in os.path.basename(obj): continue
        sass = subprocess.run(['cuobjdump', '-sass', obj], capture_output=True, text=True).stdout
        kernels, cur = collections.OrderedDict(), None
        for line in sass.split('\n'):
            m = re.search(r'Function : (\S+)', line)
            if m: cur = m.group(1); kernels[cur] = collections.Counter(); continue
            m = re.match(r'\s+/\*[0-9a-f]+\*/\s+(?:@!?U?P\d\s+)?([A-Z0-9_.]+)', line)
            if m and cur: kernels[cur][m.group(1)] += 1
        names = demangle(list(kernels))
        rows = []
        for k, cnt in kernels.items():
            nm = short(names.get(k, k))
            if wanted and not any(w in nm for w in wanted): continue
            total = sum(cnt.values())
            def c(prefix): return sum(v for op, v in cnt.items() if op.startswith(prefix))
            rows.append((nm, total, c('LDG.E.128') + c('LDG.E.NA.128') + c('LDG.E.128.CONSTANT') * 0, c('LDG') - c('LDG.E.128') - c('LDG.E.NA.128'),
                         c('STG.E.128'), c('STG') - c('STG.E.128'), c('ATOMS'), c('RED') + c('ATOMG'), c('LDS'), c('MUFU.RCP'), c('FCHK'),
                         c('F2I'), c('UBLKCP'), c('SYNCS'), c('BAR'), c('SHFL'), c('HMMA') + c('UTC') + c('QMMA') + c('IMMA')))
        if not rows: continue
        print(f'## {os.path.basename(obj).split(".")[0]}\n')
        print('| kernel | instr | LDG.128 | LDG other | STG.128 | STG other | ATOMS | RED/ATOMG | LDS | RCP | FCHK | F2I | UBLKCP | SYNCS | BAR | SHFL | MMA |')
        print('|---|---|---|---|---|---|---|---|---|---|---|---|---|---|---|---|---|')
        for r in rows: print('| `' + r[0] + '` | ' + ' | '.join(str(v) for v in r[1:]) + ' |')
        print()


if __name__ == '__main__':
    main()
