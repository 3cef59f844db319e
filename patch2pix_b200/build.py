"""Build libp2p_b200.so in-tree with nvcc for sm_90a (cross-compiles without a GPU).

    python -m patch2pix_b200.build [--force] [--verbose]
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
OUT = os.path.join(HERE, 'libp2p_b200.so')
SOURCES = ['api.cu', 'coarse.cu', 'refine.cu', 'umma_gemm.cu', 'nc_umma.cu', 'preprocess.cu', 'verify.cu', 'pose.cu', 'degensac.cu',
           'eval.cu', 'hpatches.cu', 'overlap.cu', 'nc_stack.cu', 'topk.cu', 'relpose.cu',
           'abspose.cu', 'sfm.cu', 'keypoints.cu', 'superglue.cu']
HEADERS = ['common.cuh', 'kernels.h', 'ransac_common.cuh', 'verify_common.cuh', 'umma_gemm.h', 'umma_ptx.cuh',
           os.path.join('..', '..', 'include', 'p2p_b200.h')]
NVCC_FLAGS = ['-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-lineinfo', '-std=c++17',
              '-Xcompiler', '-fPIC,-O2,-fvisibility=hidden', '--threads', '4']
# sfm.cu rounds every product and sum on its own so that its numpy oracle reproduces it bit for bit
FILE_FLAGS = {'sfm.cu': ['-fmad=false']}


def _nvcc():
    for c in (os.environ.get('NVCC'), '/usr/local/cuda/bin/nvcc', 'nvcc'):
        if c and (os.path.isabs(c) and os.path.exists(c) or not os.path.isabs(c)):
            return c
    raise RuntimeError('nvcc not found')


def needs_build():
    if not os.path.exists(OUT):
        return True
    t = os.path.getmtime(OUT)
    deps = [os.path.join(CSRC, s) for s in SOURCES + HEADERS] + [os.path.abspath(__file__)]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    if not force and not needs_build():
        return OUT
    objs = []
    procs = []
    os.makedirs(os.path.join(HERE, 'build'), exist_ok=True)
    for s in SOURCES:
        o = os.path.join(HERE, 'build', s.replace('.cu', '.o'))
        cmd = [_nvcc()] + NVCC_FLAGS + FILE_FLAGS.get(s, []) + (['-Xptxas', '-v'] if verbose else []) + ['-c', os.path.join(CSRC, s), '-o', o]
        procs.append((s, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(o)
    failed = False
    for s, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0 or verbose:
            sys.stderr.write(f'--- nvcc {s} ---\n{out}\n')
        failed |= p.returncode != 0
    if failed:
        raise RuntimeError('nvcc failed building libp2p_b200.so')
    cmd = [_nvcc(), '-shared', '-o', OUT] + objs + ['-gencode', 'arch=compute_90a,code=sm_90a']
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError('link failed:\n' + r.stdout)
    return OUT


if __name__ == '__main__':
    print(build(force='--force' in sys.argv, verbose='--verbose' in sys.argv))
