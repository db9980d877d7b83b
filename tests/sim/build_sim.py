"""Build tests/sim/libccb200_sim.so: the product kernel sources compiled by g++ against the CPU
execution-model simulator (cusim.h).  TEST TOOL ONLY - lets the GPU-less container check kernel
indexing / reductions against the oracle.  The wgmma tensor-core kernels are excluded (CCB_CPU_SIM)."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
CSRC = os.path.join(ROOT, 'cc_b200', 'csrc')
OUT = os.path.join(HERE, 'libccb200_sim.so')
SIM_SOURCES = ['common.cu', 'photo.cu', 'warp_ops.cu', 'smooth_bce.cu', 'conv_ffma.cu', 'conv_tc.cu', 'wprep.cu', 'misc_ops.cu', 'b2f_ops.cu', 'io_ops.cu']


def build(force=False):
    srcs = [os.path.join(CSRC, s) for s in SIM_SOURCES if os.path.exists(os.path.join(CSRC, s))]
    deps = srcs + [os.path.join(HERE, 'cusim.h'), os.path.join(HERE, 'cusim.cpp'),
                   os.path.join(ROOT, 'include', 'ccb200.h')] + \
        [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith('.cuh')]
    if not force and os.path.exists(OUT) and all(os.path.getmtime(OUT) > os.path.getmtime(d) for d in deps):
        return OUT
    objs = []
    bdir = os.path.join(HERE, 'build')
    os.makedirs(bdir, exist_ok=True)
    procs = []
    for s in srcs + [os.path.join(HERE, 'cusim.cpp')]:
        o = os.path.join(bdir, os.path.basename(s) + '.o')
        objs.append(o)
        cmd = ['g++', '-x', 'c++', '-std=c++17', '-O2', '-fPIC', '-DCCB_CPU_SIM', '-mfma', '-ffp-contract=off',
               '-I', HERE, '-I', CSRC, '-Wno-unused-function', '-c', s, '-o', o]
        procs.append((s, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
    for s, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            sys.stderr.write(out.decode())
            raise RuntimeError('sim build failed: ' + s)
    subprocess.check_call(['g++', '-shared', '-o', OUT] + objs)
    return OUT


if __name__ == '__main__':
    print(build(force='-f' in sys.argv))
