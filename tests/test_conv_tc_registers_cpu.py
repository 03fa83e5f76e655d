"""The convolution kernel's MMA warpgroups keep both accumulators and the fp32 total in registers: every
conv_tc_kernel instantiation (3x3 / 1x1, 3xTF32 / FP16) compiles for sm_90a with no spill stores or loads.  A spill
there puts the per-step promotion (tot += d) through local memory on every (chunk, tap) step.  nvcc cross-compiles
without a GPU, so this runs on any build machine."""
import os
import re
import subprocess

from tests.conftest import ROOT


def test_conv_tc_kernel_does_not_spill(tmp_path):
    import __graft_entry__ as ge
    nvcc = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
    src = os.path.join(ge.CSRC, 'conv_tc.cu')
    cmd = [nvcc] + ge.NVCC_FLAGS + ['-Xptxas', '-v', '-c', '-o', str(tmp_path / 'conv_tc.o'), src]
    res = subprocess.run(cmd, capture_output=True, text=True, cwd=ROOT)
    assert res.returncode == 0, res.stderr
    # ptxas prints, per entry function: "Compiling entry function '<name>'", "Function properties for <name>",
    # "<n> bytes stack frame, <s> bytes spill stores, <l> bytes spill loads"
    props = re.findall(r"Function properties for (\S+)\s*\n\s*\d+ bytes stack frame, (\d+) bytes spill stores, "
                       r"(\d+) bytes spill loads", res.stderr)
    kernels = {name: (int(st), int(ld)) for name, st, ld in props if 'conv_tc_kernel' in name}
    assert len(kernels) == 4, f'expected the four conv_tc_kernel instantiations, ptxas reported {sorted(kernels)}'
    spilling = {name: v for name, v in kernels.items() if v != (0, 0)}
    assert not spilling, f'conv_tc_kernel spills (stores, loads in bytes): {spilling}'
