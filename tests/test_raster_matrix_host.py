"""CPU: the raster-kernel coverage table of tests/test_raster_matrix_gpu.py lists every raster kernel the dispatcher of
csrc/dbw_render.cu launches, and nothing else.  A new template instantiation or kernel in the dispatcher fails here until the
GPU matrix has a case for it (which its profiler test then checks really reaches the kernel)."""
import os
import re

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, '..', 'differentiable-blocksworld_b200', 'csrc', 'dbw_render.cu')


def dispatched_raster_kernels(src):
    """template-ids `raster_*_kernel<...>` and plain `raster_*_kernel<<<` launches of the CUDA source, comments removed, with
    launch_forward's block size NT resolved to the `launch_forward<X>` arguments and X to its #define"""
    code = re.sub(r'//[^\n]*|/\*.*?\*/', '', src, flags=re.S)
    defines = dict(re.findall(r'#define\s+(\w+)\s+(\d+)\b', code))
    nts = [defines.get(x, x) for x in re.findall(r'launch_forward<(\w+)>\s*\(', code)]
    out = set()
    for name, args in re.findall(r'\b(raster_\w+_kernel)<([^<>]+)>(?!>)', code):
        args = [a.strip() for a in args.split(',')]
        for nt in (nts if 'NT' in args else [None]):
            out.add(f'{name}<{", ".join(nt if a == "NT" else a for a in args)}>')
    out |= set(re.findall(r'\b(raster_\w+_kernel)<<<', code))
    return out


def test_dispatcher_parse_finds_the_known_kernels():
    found = dispatched_raster_kernels(open(SRC).read())
    assert {'raster_hard_forward_kernel', 'raster_forward_kernel<256, true>', 'raster_forward_kernel<128, false>',
            'raster_backward_kernel<true, true, true>', 'raster_bary_backward_kernel<false>'} <= found, found


def test_every_dispatched_raster_kernel_has_a_coverage_case():
    from tests import test_raster_matrix_gpu as M           # importable without a GPU
    found = dispatched_raster_kernels(open(SRC).read())
    assert found == set(M.COVERAGE), (f'launched but not covered: {sorted(found - set(M.COVERAGE))}; '
                                      f'covered but not launched: {sorted(set(M.COVERAGE) - found)}')
    for kernel, (kind, arg) in M.COVERAGE.items():
        assert (kind == 'matrix' and arg in M.MATRIX) or (kind == 'epilogue' and isinstance(arg, int)), kernel
