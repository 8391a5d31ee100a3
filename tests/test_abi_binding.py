"""The ctypes binding against include/sgs_abi.h (no GPU): the Structure and dtype mirrors have the compiler's layout, every prototype is
typed from the header, and ctypes rejects an argument of the wrong type before the call reaches the library."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from pysgs import binding as B

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INCLUDE = os.path.join(ROOT, 'include')

# Python mirror -> C struct it restates
STRUCTS = {B.OrbParams: 'sgs_orb_params', B.Settings: 'sgs_settings', B.FrameView: 'sgs_frame_view', B.Camera: 'sgs_camera',
           B.LastFrameBatch: 'sgs_lastframe_batch', B.PoseOptBatch: 'sgs_poseopt_batch', B.PoseChainBatch: 'sgs_posechain_batch',
           B.FuseBatch: 'sgs_fuse_batch', B.InitBatch: 'sgs_init_batch', B.BowBatch: 'sgs_bow_batch', B.FrustumBatch: 'sgs_frustum_batch',
           B.LocalMapBatch: 'sgs_localmap_batch', B.KeyFrameBatch: 'sgs_keyframe_batch'}
# numpy dtype -> (C struct, C member of each dtype field where the names differ)
DTYPES = {'KP_DTYPE': (B.KP_DTYPE, 'sgs_keypoint', {}), 'OBJ_DTYPE': (B.OBJ_DTYPE, 'sgs_object2d', {k: 'rect.' + k for k in 'xywh'})}

KINDS = {C.c_int32: 'i32', C.c_int64: 'i64', C.c_uint8: 'u8', C.c_uint64: 'u64', C.c_float: 'f32', C.c_double: 'f64', C.c_void_p: 'ptr'}
NP_KINDS = {np.dtype('<i4'): 'i32', np.dtype('<f4'): 'f32'}
LAYOUT_C = r'''#include <stddef.h>
#include <stdio.h>
#include "sgs_abi.h"
#define KIND(x) _Generic((x), int32_t: "i32", int64_t: "i64", uint8_t: "u8", uint64_t: "u64", float: "f32", double: "f64", \
    default: __builtin_classify_type(x) == 5 ? "ptr" : __builtin_classify_type(x) == 12 ? "struct" : "other")
#define SIZE(py, T) { printf("%s sizeof 0 %zu struct\n", py, sizeof(T)); }
#define FIELD(py, T, name, m, e) { static T s; printf("%s %s %zu %zu %s\n", py, name, offsetof(T, m), sizeof(s.m), KIND(s.e)); }
int main(void) {
'''


def _kind(t):
    """Kind of a ctypes field type, as the C side reports it: arrays by their element."""
    if issubclass(t, C.Array):
        return _kind(t._type_)
    return 'struct' if issubclass(t, C.Structure) else KINDS[t]


def test_mirrors_match_the_compiler_layout(tmp_path):
    src, want = [LAYOUT_C], {}
    for cls, cname in STRUCTS.items():
        py = cls.__name__
        src.append('SIZE("%s", %s)' % (py, cname))
        want[py, 'sizeof'] = (0, C.sizeof(cls), 'struct')
        for name, t in cls._fields_:
            src.append('FIELD("%s", %s, "%s", %s, %s)' % (py, cname, name, name, name + '[0]' if issubclass(t, C.Array) else name))
            want[py, name] = (getattr(cls, name).offset, getattr(cls, name).size, _kind(t))
    for py, (dt, cname, member) in DTYPES.items():
        src.append('SIZE("%s", %s)' % (py, cname))
        want[py, 'sizeof'] = (0, dt.itemsize, 'struct')
        for name, (ft, off) in dt.fields.items():
            m = member.get(name, name)
            src.append('FIELD("%s", %s, "%s", %s, %s)' % (py, cname, name, m, m))
            want[py, name] = (off, ft.itemsize, NP_KINDS[ft])
    (tmp_path / 'layout.c').write_text('\n'.join(src) + '\nreturn 0; }\n')
    cc = subprocess.run(['cc', '-std=c11', '-I', INCLUDE, '-o', str(tmp_path / 'layout'), str(tmp_path / 'layout.c')], capture_output=True, text=True)
    assert cc.returncode == 0, cc.stderr
    got = {}
    for line in subprocess.check_output([str(tmp_path / 'layout')], text=True).splitlines():
        py, name, off, size, kind = line.split()
        got[py, name] = (int(off), int(size), kind)
    assert got.keys() == want.keys()
    bad = ['%s.%s: Python (offset, size, kind) %s, C %s' % (py, name, want[py, name], got[py, name]) for py, name in want if want[py, name] != got[py, name]]
    assert not bad, '\n'.join(bad)


P, S, I32, I64, Z, F32, F64 = C.c_void_p, C.c_char_p, C.c_int32, C.c_int64, C.c_size_t, C.c_float, C.c_double
PINNED = {
    'sgs_tracker_detect_device': (C.c_int, [P, P, P, I64, I32, I32, I32, I32, P]),
    'sgs_tracker_step': (C.c_int, [P, P, P, Z, I32, P, Z, I32, I32] + [P] * 10 + [F32, I32, I32] + [P] * 9),
    'sgs_extract_batch': (C.c_int, [P, P, I32, Z, I32, P, P, I32, P]),
    'sgs_fundamental_ransac': (C.c_int, [P, P, I32, F64, F64, I32, P, P, P, I32]),
    'sgs_detector_create': (C.c_int, [S, S, I32, F32, F32, I32, I32, P]),
    'sgs_last_error': (C.c_char_p, []),
    'sgs_tracker_extractor': (C.c_void_p, [P]),
    'sgs_tracker_lk': (C.c_void_p, [P]),
    'sgs_extractor_stream': (C.c_void_p, [P]),
    'sgs_extractor_destroy': (None, [P]),
}


def test_signatures_are_typed_from_the_header():
    L = B.lib()
    for name, (restype, argtypes) in PINNED.items():
        assert B._SIGNATURES[name] == (restype, argtypes), name
        assert (getattr(L, name).restype, getattr(L, name).argtypes) == (restype, argtypes), name
    by_value = {t for _, args in B._SIGNATURES.values() for t in args if t not in (P, S)}
    assert by_value == set(B._BY_VALUE.values())          # every mapped by-value type is in use, nothing else is


@pytest.mark.parametrize('proto', ['SGS_API int sgs_x(long n);', 'SGS_API int sgs_x(unsigned n);', 'SGS_API int sgs_x(uint32_t n);',
                                   'SGS_API int sgs_x(sgs_camera cam);', 'SGS_API float sgs_x(void);', 'SGS_API sgs_camera sgs_x(int n);'])
def test_an_unmapped_type_is_refused(proto):
    with pytest.raises(TypeError, match='sgs_x'):
        B.parse_abi('/* SGS_API int sgs_y(long n); */\n' + proto)


def test_an_unparsed_prototype_is_refused():
    with pytest.raises(ValueError):
        B.parse_abi('SGS_API int sgs_x(int n);\nSGS_API int (*sgs_y)(int n);')


def test_typed_names_are_the_exported_symbols():
    out = subprocess.check_output(['nm', '-D', '--defined-only', B.build()], text=True)
    assert sorted(l.split()[-1] for l in out.splitlines() if ' T ' in l and l.split()[-1].startswith('sgs_')) == B.ABI_SYMBOLS


def test_wrong_argument_types_are_rejected_before_the_call():
    L = B.lib()
    with pytest.raises(C.ArgumentError):
        L.sgs_extractor_level_info(None, 1.5, None, None, None)        # float for int
    with pytest.raises(C.ArgumentError):
        L.sgs_settings_load('settings.yaml', None)                    # str for const char*
    with pytest.raises(C.ArgumentError):
        L.sgs_detector_describe(None, None, C.c_size_t(16), None)     # size_t for int64_t
