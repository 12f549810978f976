"""Build the UNMODIFIED reference CUDA extension (`monarch_cuda`, csrc/flashfftconv of HazyResearch/flash-fft-conv) for
the H100, into oracle/_ref/ (git-ignored).

The reference's own setup.py asks torch for a GPU at import time (csrc/flashfftconv/setup.py:6-9) and emits PTX for
compute_80 only (:30), which an H100 would have to JIT at load (minutes).  This script compiles the same 25 sources,
with the same flags (-O3 --use_fast_math -std=c++17 and torch's CUDAExtension defines), directly to sm_90a SASS (wmma is
still legal there), from a scratch copy of the given reference checkout, and leaves only build products:

    oracle/_ref/monarch_cuda*.so     the extension
    oracle/_ref/flashfftconv/        the reference's pure-python package

It is used to (re)generate the stored reference outputs under tests/golden/ (tests/golden/make_ref_golden.py); nothing
else reads it.  No reference source enters the repository.
Usage:  python oracle/build_ref.py --reference PATH_TO_FLASH_FFT_CONV_CHECKOUT [-j JOBS]
"""
import argparse
import os
import shutil
import subprocess
import sys
import sysconfig
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, 'oracle', '_ref')


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reference', required=True, help='checkout of HazyResearch/flash-fft-conv')
    ap.add_argument('-j', type=int, default=5)
    args = ap.parse_args()
    REF = args.reference
    WORK = os.path.join(tempfile.gettempdir(), 'bffc_ref_build')
    import torch
    from torch.utils import cpp_extension as ce
    os.makedirs(OUT, exist_ok=True)
    if os.path.isdir(WORK):
        shutil.rmtree(WORK)
    shutil.copytree(os.path.join(REF, 'csrc', 'flashfftconv'), WORK)
    srcs = ['monarch.cpp'] + sorted(
        os.path.join(d, f) for d in ('monarch_cuda', 'butterfly', 'conv1d')
        for f in os.listdir(os.path.join(WORK, d)) if f.endswith('.cu'))
    inc = []
    for p in ce.include_paths('cuda'):
        inc += ['-I', p]
    inc += ['-I', sysconfig.get_paths()['include']]
    defs = ['-DTORCH_EXTENSION_NAME=monarch_cuda', '-DTORCH_API_INCLUDE_EXTENSION_H', '-D_GLIBCXX_USE_CXX11_ABI=1']
    nvcc_flags = ['-O3', '-lineinfo', '--use_fast_math', '-std=c++17', '--expt-relaxed-constexpr',
                  '-D__CUDA_NO_HALF_OPERATORS__', '-D__CUDA_NO_HALF_CONVERSIONS__', '-D__CUDA_NO_BFLOAT16_CONVERSIONS__',
                  '-D__CUDA_NO_HALF2_OPERATORS__', '-gencode', 'arch=compute_90a,code=sm_90a',
                  '-Xcompiler', '-fPIC', '-w']
    lines = ['rule nvcc', '  command = /usr/local/cuda/bin/nvcc $flags -c $in -o $out', '  description = NVCC $in',
             'rule cxx', '  command = g++ $flags -c $in -o $out', 'rule link', '  command = g++ -shared $in -o $out $libs']
    objs = []
    for s in srcs:
        o = os.path.join(WORK, 'obj', s.replace('/', '_') + '.o')
        objs.append(o)
        if s.endswith('.cu'):
            lines += [f'build {o}: nvcc {os.path.join(WORK, s)}', '  flags = ' + ' '.join(nvcc_flags + defs + inc)]
        else:
            lines += [f'build {o}: cxx {os.path.join(WORK, s)}',
                      '  flags = ' + ' '.join(['-O3', '-std=c++17', '-fPIC', '-w'] + defs + inc)]
    so = os.path.join(OUT, 'monarch_cuda' + sysconfig.get_config_var('EXT_SUFFIX'))
    libdirs = ce.library_paths('cuda')
    libs = ' '.join(f'-L{d} -Wl,-rpath,{d}' for d in libdirs) + ' -lc10 -lc10_cuda -ltorch_cpu -ltorch_cuda -ltorch -ltorch_python -lcudart'
    lines += [f'build {so}: link ' + ' '.join(objs), f'  libs = {libs}', f'default {so}']
    os.makedirs(os.path.join(WORK, 'obj'), exist_ok=True)
    with open(os.path.join(WORK, 'build.ninja'), 'w') as f:
        f.write('\n'.join(lines) + '\n')
    rc = subprocess.call(['ninja', '-C', WORK, '-j', str(args.j)])
    if rc:
        return rc
    # the reference's pure-python package, copied as it is (its monarch_cuda import resolves to the extension above)
    dst = os.path.join(OUT, 'flashfftconv')
    if os.path.isdir(dst):
        shutil.rmtree(dst)
    shutil.copytree(os.path.join(REF, 'flashfftconv'), dst)
    print('built', so)
    return 0


if __name__ == '__main__':
    sys.exit(main())
