"""The RPN target kernels (csrc/bags_anchor_target.cu, a translation unit of its own linked into the library) fit their
registers: ptxas's report on that unit, read with tests/ptxas_report.parse, has exactly the gt max, assign, select and
write kernels, none spills and no wgmma is serialised.  A compile of that one unit, a few seconds."""
import os
import subprocess
import tempfile

import pytest

import ptxas_report
from balancedgroupsoftmax_b200 import build as B


@pytest.fixture(scope='module')
def report():
    try:
        nvcc = B._nvcc()
    except RuntimeError:
        pytest.skip('nvcc not found')
    with tempfile.TemporaryDirectory() as tmp:
        cmd = [nvcc, '-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-std=c++17', '-cubin', '-Xptxas', '-v',
               '-o', os.path.join(tmp, 'bags_anchor_target.cubin'), os.path.join(B.CSRC, 'bags_anchor_target.cu')]
        res = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert res.returncode == 0, res.stdout
    return ptxas_report.parse(res.stdout)


def test_unit_is_linked_into_the_library():
    assert os.path.join(B.CSRC, 'bags_anchor_target.cu') in B.UNITS
    for h in ('bags_anchor_target.cuh', 'bags_anchor.cuh', 'bags_hash.cuh', 'bags_iou.cuh'):
        assert os.path.join(B.CSRC, h) in B.HEADERS, h
    assert os.path.join(B.CSRC, 'bags_anchor_target.cu') not in B.SOURCES


def test_anchor_target_kernels_do_not_spill(report):
    names = ('gt_max', 'assign', 'select', 'write')
    kernels = sorted(n for n in report if 'bags_at_' in n and '_kernel' in n)
    assert len(kernels) == 4 and all(any('bags_at_%s_kernel' % k in n for n in kernels) for k in names), kernels
    assert set(report) == set(kernels), 'entry functions other than the four kernels: %s' % sorted(report)
    bad = {n: r for n, r in report.items() if r != (0, 0, False)}
    assert not bad, '(spill store bytes, spill load bytes, wgmma serialised): %s' % bad
