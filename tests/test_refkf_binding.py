"""The ctypes mirror of sgs_refkf_batch has the compiler's layout, and the new entry points are typed from the header (no GPU)."""
import ctypes as C
import subprocess

from pysgs import binding as B
from test_abi_binding import INCLUDE, LAYOUT_C, _kind


def test_refkf_batch_mirror_matches_the_compiler_layout(tmp_path):
    cls, cname = B.RefKfBatch, 'sgs_refkf_batch'
    src = [LAYOUT_C, 'SIZE("RefKfBatch", %s)' % cname]
    want = {'sizeof': (0, C.sizeof(cls), 'struct')}
    for name, t in cls._fields_:
        src.append('FIELD("RefKfBatch", %s, "%s", %s, %s)' % (cname, name, name, name + '[0]' if issubclass(t, C.Array) else name))
        want[name] = (getattr(cls, name).offset, getattr(cls, name).size, _kind(t))
    (tmp_path / 'layout.c').write_text('\n'.join(src) + '\nreturn 0; }\n')
    cc = subprocess.run(['cc', '-std=c11', '-I', INCLUDE, '-o', str(tmp_path / 'layout'), str(tmp_path / 'layout.c')], capture_output=True, text=True)
    assert cc.returncode == 0, cc.stderr
    got = {}
    for line in subprocess.check_output([str(tmp_path / 'layout')], text=True).splitlines():
        _, name, off, size, kind = line.split()
        got[name] = (int(off), int(size), kind)
    assert got == want


def test_new_entry_points_are_typed():
    P = C.c_void_p
    L = B.lib()
    assert L.sgs_tracker_refkf_chain_device.argtypes == [P, P, P, C.c_int32, P] and L.sgs_tracker_refkf_chain_device.restype == C.c_int
    assert L.sgs_tracker_motion_discards_device.argtypes == [P, P]
    assert B.lib().sgs_tracker_motion_discards_device(None, None) == B.SGS_ERR_INVALID
