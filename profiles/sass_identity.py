"""Compare the SASS of every kernel of a base revision with the same kernel of the working tree, instruction for instruction.

    python profiles/sass_identity.py [--base REV] [--src fmpm_forward.cu ...]

Both trees are compiled to cubins with the library's own flags (fluidlab_b200/csrc/build.py) and disassembled with `cuobjdump -sass`.  Per
kernel (mangled name) the instruction text is compared after masking what legitimately moves when the kernel parameter block grows at its
end: constant-bank offsets (`c[0x0][0x...]`) and the encoding comments.  A kernel of the base that is missing from the working tree, or whose
masked instructions differ, is reported and the script exits non-zero.  Kernels that exist only in the working tree are listed as new.
Needs nvcc / cuobjdump, no GPU.
"""
import argparse
import importlib.util
import os
import re
import shutil
import subprocess
import sys
import tempfile
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC_REL = os.path.join('fluidlab_b200', 'csrc')
_spec = importlib.util.spec_from_file_location('_fmpm_build', os.path.join(ROOT, CSRC_REL, 'build.py'))
BUILD = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(BUILD)
SRCS = ['fmpm_forward.cu', 'fmpm_backward.cu', 'fmpm_io.cu', 'fmpm_rigid.cu']


def _tool(name):
    p = os.path.join(os.path.dirname(BUILD.NVCC), name)
    return p if os.path.exists(p) else shutil.which(name)


def cubin(tree, src, out_dir):
    out = os.path.join(out_dir, src + '.cubin')
    cmd = [_tool('nvcc')] + BUILD.FLAGS + ['-cubin', os.path.join(tree, CSRC_REL, src), '-o', out]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(r.stdout + r.stderr)
    return out


_FUNC = re.compile(r'^\s+Function : (\S+)')
_ANON = re.compile(r'_GLOBAL__N__[0-9a-f]+_')   # the anonymous-namespace tag hashes the source path
_INSN = re.compile(r'^\s+/\*[0-9a-f]{4,}\*/\s+(.*?)\s*;')
_CBANK = re.compile(r'c\[0x[0-9a-f]+\]\[0x[0-9a-f]+\]')


def sass(path):
    """{mangled kernel: [masked instruction text]}"""
    txt = subprocess.run([_tool('cuobjdump'), '-sass', path], capture_output=True, text=True, check=True).stdout
    out, cur = {}, None
    for line in txt.splitlines():
        m = _FUNC.match(line)
        if m:
            cur = out.setdefault(_ANON.sub('_GLOBAL__N__', m.group(1)), [])
            continue
        m = _INSN.match(line)
        if m and cur is not None:
            cur.append(_CBANK.sub('c[..][..]', m.group(1)))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--base', default='HEAD', help='git revision to compare against (default HEAD)')
    ap.add_argument('--src', nargs='*', default=SRCS)
    a = ap.parse_args()
    with tempfile.TemporaryDirectory() as tmp:
        base = os.path.join(tmp, 'base')
        os.makedirs(base)
        arc = subprocess.run(['git', '-C', ROOT, 'archive', a.base], capture_output=True, check=True).stdout
        subprocess.run(['tar', '-x', '-C', base], input=arc, check=True)
        jobs = [(t, s, os.path.join(tmp, n)) for n, t in (('b', base), ('w', ROOT)) for s in a.src]
        for _, _, d in jobs:
            os.makedirs(d, exist_ok=True)
        with ThreadPoolExecutor(4) as ex:
            cubins = list(ex.map(lambda j: cubin(*j), jobs))
        bad, n_same, new = [], 0, []
        for i, src in enumerate(a.src):
            old, cur = sass(cubins[i]), sass(cubins[len(a.src) + i])
            for k, ins in sorted(old.items()):
                if k not in cur:
                    bad.append(f'{src}: {k} missing')
                elif cur[k] != ins:
                    d = next(j for j in range(min(len(ins), len(cur[k])) + 1) if j >= min(len(ins), len(cur[k])) or ins[j] != cur[k][j])
                    bad.append(f'{src}: {k} differs ({len(ins)} -> {len(cur[k])} instructions, first difference at {d})')
                else:
                    n_same += 1
            new += [f'{src}: {k} ({len(cur[k])} instructions)' for k in sorted(set(cur) - set(old))]
    print(f'{n_same} kernels of {a.base} identical (constant-bank offsets masked)')
    for line in new:
        print('new  ', line)
    for line in bad:
        print('DIFF ', line)
    sys.exit(1 if bad else 0)


if __name__ == '__main__':
    main()
