"""CPU: the C-ABI library builds for sm_90a, loads, and exports every symbol include/hmcx.h declares.
No compute call needs a GPU here: argument validation returns before any CUDA work."""
import ctypes as C
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    text = open(os.path.join(ROOT, 'include', 'hmcx.h')).read()
    text = re.sub(r'/\*.*?\*/', '', text, flags=re.S)
    return sorted(set(re.findall(r'\b(hmcx_[a-z_0-9]+)\s*\(', text)))


def test_header_symbols_exported(built_library):
    from hamiltorch_b200 import _native
    lib = _native.load_library()
    declared = _declared_symbols()
    assert 'hmcx_hmc_run' in declared and 'hmcx_leapfrog' in declared
    for name in declared:
        assert hasattr(lib, name), 'libhmcx.so does not export ' + name
    assert sorted(_native.EXPORTED_SYMBOLS) == declared, 'binding prototypes out of sync with include/hmcx.h'
    assert lib.hmcx_abi_version() == _native.ABI_VERSION


def test_library_is_sm90a(built_library):
    import shutil
    import subprocess
    cuobjdump = shutil.which('cuobjdump') or '/usr/local/cuda/bin/cuobjdump'
    if not os.path.exists(cuobjdump):
        pytest.skip('cuobjdump not available')
    out = subprocess.run([cuobjdump, '-lelf', built_library], capture_output=True, text=True).stdout
    assert 'sm_90a' in out, out


def test_invalid_arguments_are_rejected_without_cuda(built_library):
    from hamiltorch_b200 import _native as N
    lib = N.load_library()
    tgt = N.TargetStruct()
    tgt.kind, tgt.dim = 0, 8
    mass = N.MassStruct()
    rng = N.RngStruct()
    rng.mode = N.RNG_PHILOX
    nuts = N.NutsStruct()
    # ld not a multiple of 4
    rc = lib.hmcx_hmc_run(C.byref(tgt), C.byref(mass), C.byref(rng), C.byref(nuts), None, None, None,
                          1, 7, 5, 10, 0, 0, 10, None, None, None, None, None, 0, None, None)
    assert rc == N.ERR_INVALID_ARG
    # null state pointers
    rc = lib.hmcx_hmc_run(C.byref(tgt), C.byref(mass), C.byref(rng), C.byref(nuts), None, None, None,
                          1, 8, 5, 10, 0, 0, 10, None, None, None, None, None, 0, None, None)
    assert rc == N.ERR_INVALID_ARG
    # unknown target kind
    tgt.kind = 99
    rc = lib.hmcx_leapfrog(C.byref(tgt), C.byref(mass), None, None, None, 1, 8, 5, None, None, None, None, None)
    assert rc == N.ERR_UNSUPPORTED
    assert b'unsupported' in lib.hmcx_status_string(rc)
    assert lib.hmcx_status_string(0) == b'ok'


def test_ctypes_struct_layout_matches_the_c_header(tmp_path):
    """Every struct of include/hmcx.h has the same size and field offsets in the ctypes binding (compiled with gcc)."""
    import shutil
    import subprocess
    from hamiltorch_b200 import _native as N
    gcc = shutil.which('gcc')
    if gcc is None:
        pytest.skip('gcc not available')
    pairs = {'hmcx_mlp_t': N.MlpStruct, 'hmcx_target_t': N.TargetStruct, 'hmcx_mass_t': N.MassStruct,
             'hmcx_rng_t': N.RngStruct, 'hmcx_nuts_t': N.NutsStruct, 'hmcx_rmhmc_t': N.RmhmcStruct,
             'hmcx_const_metric_t': N.ConstMetricStruct, 'hmcx_sink_t': N.SinkStruct}
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "hmcx.h"', 'int main(void) {']
    for cname, cls in pairs.items():
        lines.append('printf("%s.sizeof %%zu\\n", sizeof(%s));' % (cname, cname))
        for fname, _ in cls._fields_:
            lines.append('printf("%s.%s %%zu\\n", offsetof(%s, %s));' % (cname, fname, cname, fname))
    lines += ['return 0;', '}']
    src = tmp_path / 'probe.c'
    src.write_text('\n'.join(lines))
    exe = tmp_path / 'probe'
    subprocess.check_call([gcc, '-I', os.path.join(ROOT, 'include'), str(src), '-o', str(exe)])
    got = dict(l.split() for l in subprocess.check_output([str(exe)], text=True).splitlines())
    for cname, cls in pairs.items():
        assert int(got[cname + '.sizeof']) == C.sizeof(cls), cname
        for fname, _ in cls._fields_:
            assert int(got['%s.%s' % (cname, fname)]) == getattr(cls, fname).offset, (cname, fname)
    assert N.ABI_VERSION == int(re.search(r'#define HMCX_ABI_VERSION (\d+)',
                                          open(os.path.join(ROOT, 'include', 'hmcx.h')).read()).group(1))
