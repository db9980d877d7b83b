"""The wgmma convolution kernels (conv_tc.cu) hold their accumulators, stage sums and A fragments in registers: no
instantiation of conv_tc_kernel<N> or conv_tc_wgrad_kernel<N> spills, keeps a stack frame or uses local memory, and
ptxas serializes none of their wgmma.  A spill or a serialized wgmma does not change a result, only the speed, so
this is checked from the compiled library and from ptxas' report, without a GPU."""
import os
import re
import subprocess
import tempfile

import __graft_entry__ as ge

NS = {16, 32, 64, 128}
KERNEL = re.compile(r'_ZN3ccb(?:14conv_tc_kernel|20conv_tc_wgrad_kernel)ILi(\d+)EEEvNS_\d+Tc(?:Wgrad)?ArgsE')


def _tool(name):
    return os.path.join(os.path.dirname(ge.NVCC), name)


def _by_kernel(names):
    """{('fprop' | 'wgrad', N): name} of the eight tensor-core kernels among `names`"""
    out = {}
    for n in names:
        m = KERNEL.fullmatch(n)
        if m:
            out[('wgrad' if 'wgrad' in n else 'fprop', int(m.group(1)))] = n
    assert set(out) == {(k, n) for k in ('fprop', 'wgrad') for n in NS}, sorted(out)
    return out


def test_conv_tc_kernels_keep_to_registers():
    lib = ge.build()
    usage = subprocess.run([_tool('cuobjdump'), '--dump-resource-usage', lib], check=True, stdout=subprocess.PIPE,
                           universal_newlines=True).stdout
    res = {m.group(1): (int(m.group(2)), int(m.group(3)))
           for m in re.finditer(r'Function (\S+):\s+REG:\d+ STACK:(\d+) .*?LOCAL:(\d+)', usage)}
    for key, fn in sorted(_by_kernel(res).items()):
        assert res[fn] == (0, 0), '%s %d: stack %d, local %d bytes' % (key + res[fn])
        sass = subprocess.run([_tool('cuobjdump'), '-sass', '-fun', fn, lib], check=True, stdout=subprocess.PIPE,
                              universal_newlines=True).stdout
        assert 'HGMMA' in sass, key
        spills = re.findall(r'\b(?:LDL|STL)\b', sass)
        assert not spills, '%s %d: %d local loads / stores' % (key + (len(spills),))


def test_conv_tc_ptxas_report():
    """ptxas -v, with the library's own flags: 0 spill for every instantiation, and no wgmma serialized or wait injected
    (C7510-C7519: what ptxas does when it cannot prove a wgmma's registers are left alone while it runs)"""
    with tempfile.TemporaryDirectory() as tmp:
        p = subprocess.run([ge.NVCC] + ge.FLAGS + ['-Xptxas', '-v', '-I', os.path.join(ge.ROOT, 'include'), '-c',
                            os.path.join(ge.CSRC, 'conv_tc.cu'), '-o', os.path.join(tmp, 'conv_tc.o')],
                           stdout=subprocess.PIPE, stderr=subprocess.STDOUT, universal_newlines=True)
    assert p.returncode == 0, p.stdout
    serialized = [l for l in p.stdout.splitlines() if re.search(r'\(C751\d\)', l)]
    assert not serialized, '\n'.join(serialized)
    report = {}
    for chunk in p.stdout.split('Compiling entry function ')[1:]:
        m = re.search(r'(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads', chunk)
        report[chunk.split("'")[1]] = tuple(map(int, m.groups()))
    for key, fn in sorted(_by_kernel(report).items()):
        assert report[fn] == (0, 0, 0), '%s %d: stack, spill stores, spill loads = %s' % (key + (report[fn],))
