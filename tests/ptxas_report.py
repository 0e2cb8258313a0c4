"""ptxas's resource report for the library as it ships: what every entry function spills, and whether ptxas
serialised its wgmma.

report() compiles build.SOURCES for sm_90a with ``-Xptxas -v`` once per process (about seven minutes on an 8-core
CPU machine with CUDA 12.9) and returns parse() of what ptxas printed; it skips where no nvcc is found.  A spill or a
serialised wgmma (warnings C7512 "insufficient register resources", C7518 "WG.DP in divergent path", ...) still
computes the right thing, only slower: the wgmma of a k-block run one at a time, and spilled state goes through local
memory.
"""
import functools
import os
import re
import subprocess
import tempfile

import pytest

from balancedgroupsoftmax_b200 import build as B

_SERIALISED = re.compile(r"\(C75\d\d\) Potential Performance Loss: wgmma.*'([^']+)'")
_FUNCTION = re.compile(r'Function properties for (\S+)')
_SPILLS = re.compile(r'(\d+) bytes spill stores, (\d+) bytes spill loads')


def parse(text):
    """{mangled name: (spill store bytes, spill load bytes, wgmma serialised)} for every function in ``-Xptxas -v``
    output: each ``Function properties for X`` line, the spill line that follows it, and the C75xx wgmma warnings."""
    spills, serialised, cur = {}, set(), None
    for line in text.splitlines():
        m = _SERIALISED.search(line)
        if m:
            serialised.add(m.group(1))
            continue
        m = _FUNCTION.search(line)
        if m:
            cur = m.group(1)
            continue
        m = _SPILLS.search(line)
        if m and cur is not None:
            spills[cur] = (int(m.group(1)), int(m.group(2)))
            cur = None
    return {name: (st, ld, name in serialised) for name, (st, ld) in spills.items()}


@functools.lru_cache(maxsize=None)
def report():
    """parse() of ptxas's report on the library's sources, compiled once per process."""
    try:
        nvcc = B._nvcc()
    except RuntimeError:
        pytest.skip('nvcc not found')
    with tempfile.TemporaryDirectory() as tmp:
        cmd = [nvcc, '-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-std=c++17', '-cubin', '-Xptxas', '-v',
               '-o', os.path.join(tmp, 'bags_api.cubin')] + B.SOURCES
        res = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert res.returncode == 0, res.stdout
    return parse(res.stdout)
