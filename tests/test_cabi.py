"""CPU: the C-ABI shared library loads without a GPU and exports every symbol include/dbw_render.h declares; the
ctypes mirror of DbwRenderSettings has the C layout; argument validation fails loudly (no compute is launched)."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header_functions():
    src = open(os.path.join(ROOT, 'include', 'dbw_render.h')).read()
    src = re.sub(r'/\*.*?\*/', '', src, flags=re.S)
    return sorted(set(re.findall(r'\b(dbw_[a-z_0-9]+)\s*\(', src)))


def test_library_exports_every_declared_symbol():
    from dbw_b200 import _lib
    L = _lib.lib()
    names = _header_functions()
    assert len(names) >= 10
    for n in names:
        assert hasattr(L, n), f'{n} declared in include/dbw_render.h but not exported'
    assert set(_lib.EXPORTS) == set(names)
    assert L.dbw_abi_version() == _lib.ABI_VERSION == 8


def test_settings_struct_layout_and_workspace_query():
    from dbw_b200 import _lib
    from dbw_b200.renderer import make_settings
    assert ctypes.sizeof(_lib.DbwRenderSettings) == _lib.lib().dbw_sizeof_settings() == 29 * 4 + 4 + 8       # 29 int32/float fields, padding, one pointer
    assert ctypes.sizeof(_lib.DbwMapDesc) == 16
    s = make_settings(49, 400, 400, 10, 420, 800, 10, 0, (4.8, 4.8, 0., 0.), 1e-4, 9.21e-4, 0.001, (0, 0, 0),
                      n_map_floats=10 * 256 * 279 * 3)
    fwd, bwd = ctypes.c_size_t(0), ctypes.c_size_t(0)
    assert _lib.lib().dbw_workspace_bytes(ctypes.byref(s), ctypes.byref(fwd), ctypes.byref(bwd)) == 0
    # verts_ndc + bbox (16 B) + rec (64 B) + conv (36 B) per slot, 2F slots per view
    assert fwd.value >= 49 * (420 * 12 + 1600 * (16 + 96 + 36)) + 10 * 256 * 279 * 16
    assert bwd.value >= 49 * (1600 * 72 + 420 * 12) + 10 * 256 * 279 * 16


def test_invalid_arguments_fail_loudly_without_a_gpu():
    from dbw_b200 import _lib
    from dbw_b200.renderer import make_settings
    L = _lib.lib()
    s = make_settings(1, 8, 8, 100, 3, 1, 1, 0, (1, 1, 0, 0), 0., 0., None, (0, 0, 0))      # K = 100 > 64
    rc = L.dbw_render_forward(ctypes.byref(s), *([None] * 12), 0, None, None, None)
    assert rc != 0 and b'faces_per_pixel' in L.dbw_last_error()
    s = make_settings(1, 8, 8, 4, 3, 1, 1, 0, (1, 1, 0, 0), 0., 0., None, (0, 0, 0), n_map_floats=12)
    rc = L.dbw_render_forward(ctypes.byref(s), *([None] * 12), 0, None, None, None)
    assert rc != 0 and b'null pointer' in L.dbw_last_error()


def test_product_never_imports_the_oracle():
    pkg = os.path.join(ROOT, 'differentiable-blocksworld_b200')
    for fn in os.listdir(pkg):
        if fn.endswith('.py'):
            src = open(os.path.join(pkg, fn)).read()
            assert 'oracle' not in re.sub(r'#.*', '', src).replace('oracle_', ''), fn


def test_renderer_refuses_cpu_tensors():
    import torch
    from dbw_b200 import render_scene
    from dbw_b200._lib import DbwError
    v = torch.zeros(3, 3)
    with pytest.raises(DbwError):
        render_scene(v, torch.zeros(1, 3, dtype=torch.int32), torch.zeros(1, 3, 2), torch.zeros(1, dtype=torch.int32),
                     torch.zeros(12), [(0, 2, 2)], torch.eye(3)[None], torch.zeros(1, 3), (1, 1, 0, 0), (8, 8), 1e-4, 4)


def test_ctypes_mirrors_have_the_layout_the_c_compiler_gives_the_header(tmp_path):
    """every struct of include/dbw_render.h: size and field offsets as gcc lays them out == the ctypes mirrors in _lib.py
    (the header is plain C: it must also compile as C, not only as CUDA C++)"""
    import shutil
    import subprocess
    from dbw_b200 import _lib
    gcc = '/usr/bin/gcc' if os.path.exists('/usr/bin/gcc') else shutil.which('gcc')
    if gcc is None:
        pytest.skip('no C compiler')
    structs = {'DbwRenderSettings': _lib.DbwRenderSettings, 'DbwMapDesc': _lib.DbwMapDesc,
               'DbwSceneGeometry': _lib.DbwSceneGeometry, 'DbwLossEpilogue': _lib.DbwLossEpilogue}
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "dbw_render.h"', 'int main(void) {']
    for name, cls in structs.items():
        lines.append(f'  printf("{name} %zu\\n", sizeof({name}));')
        for field, _ in cls._fields_:
            lines.append(f'  printf("{name}.{field} %zu\\n", offsetof({name}, {field}));')
    lines += ['  return 0;', '}']
    src = tmp_path / 'layout.c'
    src.write_text('\n'.join(lines))
    exe = tmp_path / 'layout'
    subprocess.run([gcc, '-std=c99', '-Wall', '-Werror', '-I', os.path.join(ROOT, 'include'), str(src), '-o', str(exe)], check=True)
    got = dict(l.split() for l in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines())
    for name, cls in structs.items():
        assert int(got[name]) == ctypes.sizeof(cls), name
        for field, _ in cls._fields_:
            assert int(got[f'{name}.{field}']) == getattr(cls, field).offset, f'{name}.{field}'
