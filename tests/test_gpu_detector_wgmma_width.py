"""Full-width wgmma in the detector's 1x1-convolution GEMM (conv1x1_tc.cuh).  A tile of NT output channels issues each split term of a k-step
(lo*hi, hi*lo, hi*hi) as one m64n(NT)k8 wgmma instead of NT / 32 m64n32k8 ones.  Every output element sees the same products in the same order
either way, and the outputs must keep their bits:
- the probe (sg-slam_b200/probes/wgmma_width_probe.cu, built by build()) runs both issue orders on the same operands for every tile width the
  planner can choose, 32 to 256 channels, and compares the accumulators bit for bit (GPU);
- every plan of the reference model at the flagship batch names the wgmma shape its launch uses, one per tile width (CPU);
- the wide instances of the kernel do not spill and issue their wgmma at the tile's width (CPU, from the build's ptxas log and SASS)."""
import os
import re
import shutil
import subprocess

import pytest

import detector_model as DM
from pysgs import binding as B

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, 'sg-slam_b200', 'lib')
PROBE = os.path.join(LIB, 'wgmma_width_probe')
REAL = os.path.join(ROOT, 'oracle', '_ref', 'ncnn_model', 'mobilenetv3_ssdlite_voc')
WIDTHS = list(range(32, 257, 32))
KERNEL = re.compile(r'_ZN3sgs2tc17conv1x1_tc_kernelI\w+?ELi(16|32)ELi(\d)EEEv\w*')


@pytest.mark.gpu
def test_full_width_wgmma_rounds_like_the_32_channel_chunks():
    assert os.path.exists(PROBE), 'build() makes sg-slam_b200/lib/wgmma_width_probe'
    r = subprocess.run([PROBE], capture_output=True, text=True, timeout=300)
    print(r.stdout)
    rows = {int(m.group(1)): m for m in re.finditer(r'^N=(\d+) elements=(\d+) differing=(\d+) zeros=(\d+) subnormal=(\d+) max_err_over_S=(\S+) (ok|FAIL)$',
                                                    r.stdout, re.M)}
    assert sorted(rows) == WIDTHS, r.stdout + r.stderr
    for n, m in rows.items():
        assert int(m.group(3)) == 0, 'N=%d: %s of %s accumulators differ' % (n, m.group(3), m.group(2))
        assert m.group(7) == 'ok', m.group(0)
    assert r.returncode == 0, r.stdout + r.stderr


def _plans(pp, bp, frames):
    d = B.Detector(pp, bp, max_frames=frames, flags=B.DET_PLAN_ONLY)
    try:
        return DM.parse_plan(d.describe())
    finally:
        d.close()


def _check_shapes(plans):
    for p in plans:
        m = re.search(r' wgmma m64n(\d+)k8', p['line'])
        assert m and int(m.group(1)) == p['nt'] and p['nt'] in WIDTHS, p['line']


@pytest.mark.skipif(not os.path.exists(REAL + '.param'), reason='reference model copy (oracle/_ref/ncnn_model, made by build()) not present')
def test_every_plan_of_the_reference_model_issues_its_tile_width():
    plans = _plans(REAL + '.param', REAL + '.bin', 512)
    assert len(plans) == 66
    _check_shapes(plans)
    assert sum(p['nt'] > 32 for p in plans) >= 20 and any(p['nt'] == 256 for p in plans)


def test_every_probe_plan_issues_its_tile_width(tmp_path):
    plans = _plans(*DM.write_probe_model(str(tmp_path), DM.GEMM_PROBES, 0)[:2], DM.PROBE_FRAMES)
    _check_shapes(plans)
    assert {p['nt'] > 32 for p in plans} == {False, True}


def _detector_object():
    obj = os.path.join(LIB, 'obj', 'detector.o')
    if not os.path.exists(obj):
        pytest.skip('sg-slam_b200/lib/obj/detector.o not built')
    return obj


def test_wide_instances_do_not_spill():
    """ptxas -v of detector.cu (kept by the Makefile): the instances of every tile width above 32 channels, for both k-block widths and every
    tail kind, have no spill stores or loads."""
    _detector_object()
    with open(os.path.join(LIB, 'obj', 'detector.ptxas.log')) as f:
        log = f.read()
    seen = set()
    for m in re.finditer(r"Function properties for (\S+)\n\s+(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", log):
        k = KERNEL.fullmatch(m.group(1))
        if not k or int(k.group(2)) < 2:
            continue
        seen.add((int(k.group(1)), int(k.group(2))))
        assert m.group(3) == m.group(4) == '0', m.group(0)
    assert seen == {(bk, c) for bk in (16, 32) for c in range(2, 9)}, seen


def test_wide_instances_issue_full_width_hgmma():
    obj = _detector_object()
    tool = shutil.which('cuobjdump') or '/usr/local/cuda/bin/cuobjdump'
    if not os.path.exists(tool):
        pytest.skip('cuobjdump not available')
    sass = subprocess.run([tool, '-sass', obj], capture_output=True, text=True, timeout=600).stdout
    per_fn = {}
    for block in re.split(r'\n\s+Function : ', sass)[1:]:
        name = block.split('\n', 1)[0].strip()
        k = KERNEL.fullmatch(name)
        if k:
            per_fn[name] = (int(k.group(2)), set(int(n) for n in re.findall(r'HGMMA\.64x(\d+)x8', block)))
    assert len(per_fn) == 8 * 2 * 8, len(per_fn)
    for name, (c, shapes) in per_fn.items():
        assert shapes == {32 * c}, (name, shapes)
