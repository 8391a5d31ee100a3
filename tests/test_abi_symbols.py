"""The C-ABI library loads and exports every symbol include/sgs_abi.h declares (no GPU, no compute calls)."""
import ctypes as C
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    txt = open(os.path.join(ROOT, 'include', 'sgs_abi.h')).read()
    return sorted(set(re.findall(r'SGS_API\s+[\w\s\*]+?\b(sgs_\w+)\s*\(', txt)))


def test_library_exports_every_declared_symbol():
    from pysgs import binding
    so = binding.build()
    lib = C.CDLL(so)
    names = _declared()
    assert len(names) >= 25
    for n in names:
        assert hasattr(lib, n), 'missing export: ' + n
    assert lib.sgs_abi_version() == 1


def test_only_abi_symbols_are_exported():
    from pysgs import binding
    out = subprocess.check_output(['nm', '-D', '--defined-only', binding.build()]).decode()
    ours = [l.split()[-1] for l in out.splitlines() if ' T ' in l and l.split()[-1].startswith('sgs_')]
    assert sorted(ours) == _declared()


def test_no_device_fails_loudly():
    """Without a CUDA device the product must fail with SGS_ERR_CUDA, never fall back to a CPU path."""
    import numpy as np
    import pytest
    from pysgs import binding
    n = C.c_int(-1)
    code = binding.lib().sgs_device_count(C.byref(n))
    if code == 0 and n.value > 0:
        pytest.skip('a CUDA device is present')
    with pytest.raises(binding.SgsError) as e:
        binding.Extractor(640, 480)
    assert e.value.code == binding.SGS_ERR_CUDA
    with pytest.raises(binding.SgsError):
        binding.hamming_bf(np.zeros((4, 32), np.uint8), np.zeros((4, 32), np.uint8))


def test_product_never_references_the_oracle():
    """oracle/ is test infrastructure: nothing under sg-slam_b200/ or include/ may import, link or mention it as a dependency."""
    bad = []
    for base in ('sg-slam_b200', 'include'):
        for dp, _, files in os.walk(os.path.join(ROOT, base)):
            for f in files:
                if f.endswith(('.so', '.o', '.log', '.pyc')):
                    continue
                txt = open(os.path.join(dp, f), errors='replace').read()
                if re.search(r'liboracle|import oracle|from oracle|oracle/|sgo_', txt):
                    # comments that merely say "never includes oracle/" are fine
                    lines = [l for l in txt.splitlines() if re.search(r'liboracle|import oracle|from oracle|oracle/|sgo_', l)
                             and 'never' not in l and 'not' not in l.lower()]
                    if lines:
                        bad.append((os.path.join(dp, f), lines[:2]))
    assert not bad, bad
