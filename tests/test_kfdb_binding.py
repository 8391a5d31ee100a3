"""The ctypes mirror of sgs_reloc_batch has the compiler's layout, and the key-frame database entry points are typed from the header (no GPU)."""
import ctypes as C
import subprocess

from pysgs import binding as B
from test_abi_binding import INCLUDE, LAYOUT_C, _kind


def test_reloc_batch_mirror_matches_the_compiler_layout(tmp_path):
    cls, cname = B.RelocBatch, 'sgs_reloc_batch'
    src = [LAYOUT_C, 'SIZE("RelocBatch", %s)' % cname]
    want = {'sizeof': (0, C.sizeof(cls), 'struct')}
    for name, t in cls._fields_:
        src.append('FIELD("RelocBatch", %s, "%s", %s, %s)' % (cname, name, name, name + '[0]' if issubclass(t, C.Array) else name))
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
    P, I = C.c_void_p, C.c_int32
    L = B.lib()
    assert L.sgs_kfdb_create.argtypes == [I, I, I, I, P]
    assert L.sgs_kfdb_add.argtypes == [P, I, P, P, P, P, P, I, P]
    assert L.sgs_kfdb_erase.argtypes == [P, I, P, P] and L.sgs_kfdb_clear.argtypes == [P, I, P]
    assert L.sgs_kfdb_reloc_candidates_device.argtypes == [P, I, P, P, P, P, I, P, P, I, P, P, P]
    assert L.sgs_bow_vector_batch_device.argtypes == [P, P, P, I, I, P, P, P, P]
    assert L.sgs_tracker_reloc_candidates_device.argtypes == [P, P, P, P, I, P] and L.sgs_tracker_reloc_candidates_device.restype == C.c_int
    # refused on the host, before any device work
    assert L.sgs_kfdb_add(None, 1, None, None, None, None, None, 1, None) == B.SGS_ERR_INVALID
    assert L.sgs_kfdb_reloc_candidates_device(None, 1, None, None, None, None, 1, None, None, 1, None, None, None) == B.SGS_ERR_INVALID
    assert L.sgs_tracker_reloc_candidates_device(None, None, None, None, 1, None) == B.SGS_ERR_INVALID
