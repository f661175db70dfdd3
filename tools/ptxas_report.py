"""Registers, spills and compiler-injected wgmma fences of every conv kernel instantiation.

Compiles cvpytorch_b200/csrc/conv_tc.cu for sm_90a with the library's flags and `-Xptxas -v` (into a temporary directory; nothing is
written to the tree) and prints one row per conv_tc_kernel instantiation: its template arguments, registers, spill store / load bytes,
the number of C7519 notes ("warpgroup.arrive is injected", a fence ptxas adds before ordinary code may touch the accumulator registers)
and the number of notes that say ptxas serialized its wgmmas (C7510, C7515, ...: every wgmma waits for the previous one, far worse).

  python tools/ptxas_report.py            # table of every instantiation ('*': a YOLOv5-s / YOLOX-s / FCOS / DeepLab plan selects it)
  python tools/ptxas_report.py --check    # exit 1 if a selected instantiation serializes, or spills / fences more than SELECTED allows
  python tools/ptxas_report.py --log F    # parse a saved `-Xptxas -v` log instead of compiling
"""
import argparse
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, 'cvpytorch_b200', 'csrc', 'conv_tc.cu')
FIELDS = ('BN', 'BK', 'F32', 'YOLO', 'EPI', 'PP', 'CTAS')

# Template arguments (BN, BK, F32, YOLO, EPI, PP, CTAS) of the instantiations the planner selects for the layers of the YOLOv5-s
# (640^2, batch 64), YOLOX-s (640^2), FCOS (800^2) and DeepLab (1024 x 2048) inference graphs at the batch sizes bench.py runs them.
# Derived by building each graph on an H100 with CVB_PLAN_DEBUG=1 (one "[cvb plan]" line per layer: block_n, block_k, fp32 output,
# fused decode, epilogue, schedule, CTAs per SM) and taking the distinct tuples.  A planner change that selects another kernel must
# extend this list.  The value is what the instantiation may still have: (spill bytes, injected fences).  (0, 0) is the goal; the
# non-zero entries are the known gaps of DESIGN.md 6 (the cooperative kernels keep the K-step predicate of the row-window stems).
SELECTED = {
    (32, 32, 0, 0, 0, 0, 2): (136, 6),
    (32, 32, 0, 0, 1, 0, 2): (0, 6),
    (32, 32, 0, 0, 3, 0, 2): (0, 6),
    (32, 32, 1, 0, 0, 0, 2): (136, 6),
    (32, 64, 0, 0, 1, 0, 1): (0, 10),
    (32, 64, 0, 0, 3, 0, 1): (0, 10),
    (32, 64, 1, 0, 0, 1, 1): (0, 0),
    (64, 32, 0, 0, 1, 0, 1): (0, 6),
    (64, 32, 0, 0, 3, 0, 1): (0, 6),
    (64, 64, 0, 0, 0, 1, 1): (0, 0),
    (64, 64, 0, 0, 1, 0, 1): (0, 10),
    (64, 64, 0, 0, 1, 1, 1): (0, 0),
    (64, 64, 0, 0, 2, 1, 1): (0, 0),
    (64, 64, 0, 0, 3, 0, 1): (0, 10),
    (64, 64, 0, 0, 3, 1, 1): (0, 0),
    (128, 32, 0, 0, 2, 0, 1): (144, 6),
    (128, 32, 1, 1, 0, 0, 1): (40, 6),
    (128, 64, 0, 0, 0, 1, 1): (1060, 0),
    (128, 64, 0, 0, 1, 1, 1): (0, 0),
    (128, 64, 0, 0, 3, 1, 1): (0, 0),
    (128, 64, 0, 0, 4, 1, 1): (0, 0),
    (128, 64, 1, 0, 0, 1, 1): (176, 0),
}


def compile_log(nvcc):
    flags = ['-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-lineinfo', '-std=c++17', '-Xcompiler', '-fPIC,-O3',
             '-I' + os.path.join(ROOT, 'include'), '-Xptxas', '-v']
    with tempfile.TemporaryDirectory() as tmp:
        r = subprocess.run([nvcc, *flags, '-c', SRC, '-o', os.path.join(tmp, 'conv_tc.o')], capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise SystemExit(f'nvcc failed ({r.returncode})')
    return r.stdout + r.stderr


def template_args(mangled):
    """conv_tc_kernel<...> template arguments from the mangled name (Li<n>E integers, Lb<0|1>E booleans), or None."""
    m = re.search(r'conv_tc_kernelI((?:L[ib]\d+E)+)EEv', mangled)
    if not m:
        return None
    return tuple(int(v) for v in re.findall(r'L[ib](\d+)E', m.group(1)))


def new_row():
    return {'regs': 0, 'st': 0, 'ld': 0, 'fence': 0, 'serial': 0}


def parse(log):
    rows = {}
    cur = None
    for line in log.splitlines():
        m = re.search(r"Compiling entry function '([^']+)'", line)
        if m:
            cur = template_args(m.group(1))
            if cur is not None:
                rows.setdefault(cur, new_row())
            continue
        m = re.search(r"\((C75\d\d)\).*function '([^']+)'", line)
        if m:
            key = template_args(m.group(2))
            if key is not None:
                col = 'fence' if m.group(1) == 'C7519' else ('serial' if 'serialized' in line else None)
                if col:
                    rows.setdefault(key, new_row())[col] += 1
            continue
        if cur is None:
            continue
        m = re.search(r'(\d+) bytes spill stores, (\d+) bytes spill loads', line)
        if m:
            rows[cur]['st'], rows[cur]['ld'] = int(m.group(1)), int(m.group(2))
        m = re.search(r'Used (\d+) registers', line)
        if m:
            rows[cur]['regs'] = int(m.group(1))
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--check', action='store_true', help='exit 1 if a selected instantiation spills or has an injected fence')
    ap.add_argument('--log', help='parse this saved ptxas -v log instead of compiling')
    ap.add_argument('--nvcc', default=os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc'))
    args = ap.parse_args()
    log = open(args.log).read() if args.log else compile_log(args.nvcc)
    rows = parse(log)
    if not rows:
        raise SystemExit('no conv_tc_kernel instantiation in the ptxas output')
    print(' '.join(f'{f:>5}' for f in FIELDS) + '   regs  spill_st  spill_ld  fences  serialized  selected')
    bad = []
    for key in sorted(rows):
        r = rows[key]
        sel = key in SELECTED
        print(' '.join(f'{v:>5}' for v in key) +
              f"   {r['regs']:>4}  {r['st']:>8}  {r['ld']:>8}  {r['fence']:>6}  {r['serial']:>10}  {'*' if sel else ''}")
        if sel:
            spill_ok, fence_ok = SELECTED[key]
            if r['serial'] or max(r['st'], r['ld']) > spill_ok or r['fence'] > fence_ok:
                bad.append(key)
    missing = sorted(set(SELECTED) - set(rows))
    n_sel = sum(k in SELECTED for k in rows)
    print(f'{len(rows)} instantiations, {n_sel} selected; spilling: {sum(1 for r in rows.values() if r["st"] or r["ld"])}, '
          f'with injected fences: {sum(1 for r in rows.values() if r["fence"])}, serialized: {sum(1 for r in rows.values() if r["serial"])}')
    if args.check:
        for key in missing:
            print('missing selected instantiation:', dict(zip(FIELDS, key)))
        for key in bad:
            print('serialized, or more spills / injected fences than recorded:', dict(zip(FIELDS, key)), rows[key])
        if bad or missing:
            return 1
    return 0


if __name__ == '__main__':
    sys.exit(main())
