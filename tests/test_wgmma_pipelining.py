"""CPU-only guard for the tensor-core kernels' code generation: compiled for sm_90a exactly as the library is, every
umma_gemm_kernel and NeighConsensus kernel instantiation keeps its wgmma chains pipelined (no ptxas "wgmma ...
serialized" advisory: C7510 function call, C7514 accumulator read by a non-wgmma instruction, C7518 warpgroup wait
in a divergent path) and spills nothing.  A serialised kernel still computes the right result, only about twice as
slowly, so the GPU parity tests cannot catch this."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KERNELS = ('umma_gemm_kernel', 'nc_l1_umma_kernel', 'nc_l2_umma_kernel')


def _ptxas_report(src, out_dir):
    from patch2pix_b200 import build as b
    nvcc = b._nvcc()
    if shutil.which(nvcc) is None:
        pytest.skip('nvcc not available')
    cmd = [nvcc] + b.NVCC_FLAGS + ['-Xptxas', '-v', '-c', os.path.join(b.CSRC, src),
                                   '-o', os.path.join(out_dir, src.replace('.cu', '.o'))]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    return r.stdout + r.stderr


@pytest.mark.parametrize('src, n_kernels', [('umma_gemm.cu', 22), ('nc_umma.cu', 5)])
def test_tensor_core_kernels_pipeline_wgmma_without_spills(tmp_path, src, n_kernels):
    log = _ptxas_report(src, str(tmp_path))
    serialised = [ln for ln in log.splitlines() if re.search(r'C75\d\d|wgmma.*serializ', ln)]
    assert not serialised, '\n'.join(serialised)
    spills, cur = {}, None
    for ln in log.splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", ln)
        if m:
            cur = m.group(1) if any(k in m.group(1) for k in KERNELS) else None
            continue
        m = re.search(r'(\d+) bytes spill stores, (\d+) bytes spill loads', ln)
        if m and cur is not None:
            spills[cur] = int(m.group(1)) + int(m.group(2))
            cur = None
    assert len(spills) == n_kernels, sorted(spills)
    assert not {k: v for k, v in spills.items() if v}, spills
