"""Build libhmcx.so in-tree with nvcc for sm_90a (H100; cross-compiles without a GPU).

    python -m hamiltorch_b200.build [--force] [--verbose]

The .so is git-ignored (history stays source-only) but is rebuilt by `__graft_entry__.build()` on every checkout.
"""
import glob
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
LIB_DIR = os.path.join(HERE, 'lib')
LIB = os.path.join(LIB_DIR, 'libhmcx.so')
LIB_FLAGS = LIB + '.flags'          # the nvcc flags (architecture included) the library was built with

NVCC_FLAGS = ['-gencode', 'arch=compute_90a,code=sm_90a', '-lineinfo', '-O3', '-std=c++17',
              '--fmad=false',          # parity arithmetic: never contract a*b+c (see hmcx_common.cuh)
              '-Xcompiler', '-fPIC']


def _nvcc():
    for cand in (os.environ.get('NVCC'), shutil.which('nvcc'), '/usr/local/cuda/bin/nvcc'):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError('nvcc not found')


def sources():
    return sorted(glob.glob(os.path.join(CSRC, '*.cu')))


def _deps():
    return sources() + glob.glob(os.path.join(CSRC, '*.cuh')) + \
        glob.glob(os.path.join(os.path.dirname(HERE), 'include', '*.h')) + [os.path.abspath(__file__)]


def _obj_of(src):
    return os.path.join(LIB_DIR, 'obj', os.path.basename(src)[:-3] + '.o')


def _flags():
    return NVCC_FLAGS + os.environ.get('HMCX_NVCC_EXTRA', '').split()


def up_to_date():
    """The library was built with the current flags (so one built for another architecture is rebuilt), it is newer
    than every source and header, and every object is newer than its source and the shared headers (a source edited
    while a build was running is therefore rebuilt next time)."""
    if not os.path.exists(LIB) or not os.path.exists(LIB_FLAGS):
        return False
    with open(LIB_FLAGS) as f:
        if f.read() != ' '.join(_flags()):
            return False
    t = os.path.getmtime(LIB)
    if not all(os.path.getmtime(f) <= t for f in _deps()):
        return False
    common = [f for f in _deps() if not f.endswith('.cu')]
    for src in sources():
        obj = _obj_of(src)
        if os.path.exists(obj) and any(os.path.getmtime(f) > os.path.getmtime(obj) for f in [src] + common):
            return False
    return True


def build(force=False, verbose=False):
    """Compile every .cu under csrc/ to one object each (in parallel) and link libhmcx.so."""
    if not force and up_to_date():
        return LIB
    os.makedirs(LIB_DIR, exist_ok=True)
    obj_dir = os.path.join(LIB_DIR, 'obj')
    os.makedirs(obj_dir, exist_ok=True)
    nvcc = _nvcc()
    procs, objs = [], []
    flags = _flags()
    stamp = ' '.join(flags)
    common = [f for f in _deps() if not f.endswith('.cu')]
    for src in sources():
        obj = os.path.join(obj_dir, os.path.basename(src)[:-3] + '.o')
        objs.append(obj)
        # per-object incremental rebuild: same flags, object newer than its source and every shared header
        flagfile = obj + '.flags'
        if (not force and os.path.exists(obj) and os.path.exists(flagfile) and open(flagfile).read() == stamp
                and all(os.path.getmtime(f) <= os.path.getmtime(obj) for f in [src] + common)):
            continue
        cmd = [nvcc] + flags + (['-Xptxas', '-v'] if verbose else []) + ['-c', src, '-o', obj]
        procs.append((src, flagfile, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    for src, flagfile, p in procs:
        out, _ = p.communicate()
        if verbose or p.returncode != 0:
            sys.stderr.write(out)
        if p.returncode != 0:
            raise RuntimeError('nvcc failed on ' + src)
        with open(flagfile, 'w') as f:
            f.write(stamp)
    tmp = LIB + '.tmp'
    subprocess.check_call([nvcc, '-shared', '-o', tmp] + objs + ['-gencode', 'arch=compute_90a,code=sm_90a'])
    os.replace(tmp, LIB)
    with open(LIB_FLAGS, 'w') as f:
        f.write(stamp)
    return LIB


if __name__ == '__main__':
    print(build(force='--force' in sys.argv, verbose='--verbose' in sys.argv))
