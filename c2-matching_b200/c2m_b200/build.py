"""Build libc2m_sm100.so in-tree with nvcc for sm_90a (cross-compiles without a GPU)."""
import os
import subprocess

PKG_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(PKG_ROOT, 'csrc')
LIB_DIR = os.path.join(PKG_ROOT, 'lib')
LIB_PATH = os.path.join(LIB_DIR, 'libc2m_sm100.so')
SOURCES = ['c_abi.cu', 'corr_aux.cu', 'corr_umma.cu', 'dcn_v2.cu', 'offsets.cu', 'conv3x3_umma.cu', 'dcn_umma.cu', 'dcn_bwd.cu',
           'psroi.cu', 'det_gather.cu', 'conv3x3_wgrad.cu', 'dcn_tc_bwd.cu']
NVCC_FLAGS = ['-gencode', 'arch=compute_90a,code=sm_90a', '-lineinfo', '-O3', '-std=c++17',
              '-shared', '-Xcompiler', '-fPIC']


def _stale():
    if not os.path.exists(LIB_PATH):
        return True
    t = os.path.getmtime(LIB_PATH)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + \
           [os.path.join(os.path.dirname(PKG_ROOT), 'include', 'c2m_sm100.h')]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    if not force and not _stale():
        return LIB_PATH
    os.makedirs(LIB_DIR, exist_ok=True)
    nvcc = os.environ.get('NVCC', 'nvcc')
    cmd = [nvcc] + NVCC_FLAGS + (['-Xptxas', '-v'] if verbose else []) + ['-o', LIB_PATH] + SOURCES
    subprocess.run(cmd, check=True, cwd=CSRC)
    return LIB_PATH


if __name__ == '__main__':
    print(build(force=True, verbose=True))
