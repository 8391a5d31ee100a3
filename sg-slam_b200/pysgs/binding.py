"""ctypes binding of libsgs_cuda.so (include/sgs_abi.h) for the Python-side harness (tests, bench).

lib() types every sgs_* function from the prototypes in sgs_abi.h, so ctypes converts the arguments (a Python float becomes a C float,
an int a size_t or int64_t) and rejects one of the wrong type before the call.

There is NO CPU fallback: loading fails loudly when the library has not been built, and every call fails with
SGS_ERR_CUDA on a machine without a CUDA device."""
import ctypes as C
import os
import re
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_PKG = os.path.dirname(_HERE)
LIB_PATH = os.path.join(_PKG, 'lib', 'libsgs_cuda.so')
_LIB = None

KP_DTYPE = np.dtype([('x', '<f4'), ('y', '<f4'), ('size', '<f4'), ('angle', '<f4'), ('response', '<f4'),
                     ('octave', '<i4'), ('class_id', '<i4')])

SGS_OK, SGS_ERR_INVALID, SGS_ERR_CUDA, SGS_ERR_CAPACITY, SGS_ERR_UNSUPPORTED = range(5)


class SgsError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__('sgs status %d: %s' % (code, msg))
        self.code = code


class OrbParams(C.Structure):
    _fields_ = [('nfeatures', C.c_int32), ('scale_factor', C.c_float), ('nlevels', C.c_int32),
                ('ini_th_fast', C.c_int32), ('min_th_fast', C.c_int32)]


class Settings(C.Structure):
    _fields_ = [(k, C.c_float) for k in ('fx', 'fy', 'cx', 'cy', 'k1', 'k2', 'p1', 'p2', 'k3', 'bf', 'fps')] + [('width', C.c_int32), ('height', C.c_int32), ('rgb', C.c_int32),
                ('th_depth', C.c_float), ('depth_map_factor', C.c_float), ('orb', OrbParams), ('detection_confidence_threshold', C.c_float),
                ('dynamic_detection_confidence_threshold', C.c_float)]


class RgbdFormat(C.Structure):          # sgs_rgbd_format
    _fields_ = [('rgb', C.c_int32), ('depth_type', C.c_int32), ('depth_map_factor', C.c_float), ('dist_coef', C.c_float * 5)]


DEPTH_U16, DEPTH_F32 = 0, 1


def rgbd_format(settings, depth_type=DEPTH_U16):
    """The sgs_rgbd_format of a loaded Settings: Camera.RGB, mDepthMapFactor and k1 k2 p1 p2 k3."""
    f = RgbdFormat(settings.rgb, depth_type, settings.depth_map_factor)
    for i, k in enumerate(('k1', 'k2', 'p1', 'p2', 'k3')):
        f.dist_coef[i] = getattr(settings, k)
    return f


class FrameView(C.Structure):
    _fields_ = [('n', C.c_int32), ('keys_un', C.c_void_p), ('u_right', C.c_void_p), ('desc', C.c_void_p),
                ('min_x', C.c_float), ('min_y', C.c_float), ('max_x', C.c_float), ('max_y', C.c_float),
                ('fx', C.c_float), ('fy', C.c_float), ('cx', C.c_float), ('cy', C.c_float), ('bf', C.c_float),
                ('nlevels', C.c_int32), ('scale_factors', C.c_void_p)]


class Camera(C.Structure):
    _fields_ = [('min_x', C.c_float), ('min_y', C.c_float), ('max_x', C.c_float), ('max_y', C.c_float),
                ('fx', C.c_float), ('fy', C.c_float), ('cx', C.c_float), ('cy', C.c_float), ('bf', C.c_float),
                ('nlevels', C.c_int32), ('scale_factors', C.c_float * 16)]


class LastFrameBatch(C.Structure):
    _fields_ = [('cam', Camera),
                ('cur_kps', C.c_void_p), ('cur_desc', C.c_void_p), ('cur_uright', C.c_void_p), ('cur_n', C.c_void_p),
                ('last_xyz', C.c_void_p), ('last_desc', C.c_void_p), ('last_flags', C.c_void_p), ('last_octave', C.c_void_p),
                ('last_angle', C.c_void_p), ('last_n', C.c_void_p), ('tcw_cur', C.c_void_p), ('tcw_last', C.c_void_p),
                ('th', C.c_float), ('mono', C.c_int32), ('check_orientation', C.c_int32),
                ('cur_mp', C.c_void_p), ('cur_mp_obs_in', C.c_void_p), ('nmatches', C.c_void_p), ('ncand', C.c_void_p), ('frame_enable', C.c_void_p)]


class KeyFrameBatch(C.Structure):
    _fields_ = [('cam', Camera),
                ('cur_kps', C.c_void_p), ('cur_desc', C.c_void_p), ('cur_uright', C.c_void_p), ('cur_n', C.c_void_p),
                ('kf_xyz', C.c_void_p), ('kf_desc', C.c_void_p), ('kf_valid', C.c_void_p), ('kf_angle', C.c_void_p),
                ('kf_min_dist', C.c_void_p), ('kf_max_dist', C.c_void_p), ('kf_n', C.c_void_p), ('tcw_cur', C.c_void_p),
                ('th', C.c_float), ('orb_dist', C.c_int32), ('check_orientation', C.c_int32),
                ('cur_mp', C.c_void_p), ('nmatches', C.c_void_p), ('ncand', C.c_void_p)]


class PoseOptBatch(C.Structure):
    _fields_ = [('cam', Camera), ('tcw_in', C.c_void_p), ('kps', C.c_void_p), ('uright', C.c_void_p), ('n', C.c_void_p), ('cap', C.c_int32),
                ('has_mp', C.c_void_p), ('mp_index', C.c_void_p), ('points_xyz', C.c_void_p), ('point_cap', C.c_int32), ('inv_level_sigma2', C.c_float * 16),
                ('tcw_out', C.c_void_p), ('outlier', C.c_void_p), ('ninliers', C.c_void_p), ('scratch_err', C.c_void_p), ('scratch_level', C.c_void_p),
                ('points2_xyz', C.c_void_p), ('id_base2', C.c_int32), ('point2_cap', C.c_int32)]


class PoseChainBatch(C.Structure):          # sgs_posechain_batch
    _fields_ = [('last_xyz', C.c_void_p), ('last_desc', C.c_void_p), ('last_flags', C.c_void_p), ('last_octave', C.c_void_p), ('last_angle', C.c_void_p),
                ('last_n', C.c_void_p), ('tcw_cur', C.c_void_p), ('tcw_last', C.c_void_p), ('th', C.c_float), ('mono', C.c_int32), ('check_orientation', C.c_int32),
                ('last_local_id', C.c_void_p),
                ('mp_xyz', C.c_void_p), ('mp_normal', C.c_void_p), ('mp_min_dist', C.c_void_p), ('mp_max_dist', C.c_void_p), ('mp_desc', C.c_void_p),
                ('mp_valid', C.c_void_p), ('mp_obs', C.c_void_p), ('mp_n', C.c_void_p), ('mp_cap', C.c_int32),
                ('th_local', C.c_float), ('nnratio_local', C.c_float), ('inv_level_sigma2', C.c_float * 16),
                ('tcw_motion', C.c_void_p), ('tcw_final', C.c_void_p), ('f_mp', C.c_void_p), ('outlier', C.c_void_p), ('stats', C.c_void_p)]


class RefKfBatch(C.Structure):              # sgs_refkf_batch
    _fields_ = [('kf_node', C.c_void_p), ('kf_weight', C.c_void_p), ('kf_desc', C.c_void_p), ('kf_angle', C.c_void_p), ('kf_xyz', C.c_void_p),
                ('kf_flags', C.c_void_p), ('kf_n', C.c_void_p), ('kf_local_id', C.c_void_p), ('tcw_last', C.c_void_p), ('frame_enable', C.c_void_p),
                ('seen_in', C.c_void_p),
                ('mp_xyz', C.c_void_p), ('mp_normal', C.c_void_p), ('mp_min_dist', C.c_void_p), ('mp_max_dist', C.c_void_p), ('mp_desc', C.c_void_p),
                ('mp_valid', C.c_void_p), ('mp_obs', C.c_void_p), ('mp_n', C.c_void_p), ('mp_cap', C.c_int32),
                ('th_local', C.c_float), ('nnratio_local', C.c_float), ('inv_level_sigma2', C.c_float * 16),
                ('tcw_refkf', C.c_void_p), ('tcw_final', C.c_void_p), ('f_mp', C.c_void_p), ('outlier', C.c_void_p), ('stats', C.c_void_p)]


class RelocBatch(C.Structure):              # sgs_reloc_batch
    _fields_ = [('map', C.c_void_p), ('frame_enable', C.c_void_p), ('covis', C.c_void_p), ('cand', C.c_void_p), ('cand_cap', C.c_int32),
                ('ncand', C.c_void_p), ('stats', C.c_void_p)]


class FuseBatch(C.Structure):
    _fields_ = [('cam', Camera), ('kf_kps', C.c_void_p), ('kf_desc', C.c_void_p), ('kf_uright', C.c_void_p), ('kf_n', C.c_void_p), ('kf_cap', C.c_int32),
                ('tcw', C.c_void_p), ('ow', C.c_void_p), ('mp_xyz', C.c_void_p), ('mp_normal', C.c_void_p), ('mp_min_dist', C.c_void_p), ('mp_max_dist', C.c_void_p),
                ('mp_desc', C.c_void_p), ('mp_valid', C.c_void_p), ('mp_n', C.c_void_p), ('mp_cap', C.c_int32), ('th', C.c_float), ('inv_level_sigma2', C.c_float * 16),
                ('sim3_variant', C.c_int32), ('xform2', C.c_void_p), ('best_idx', C.c_void_p), ('best_dist', C.c_void_p), ('kf_matched', C.c_void_p), ('nmatches', C.c_void_p)]


class InitBatch(C.Structure):
    _fields_ = [('cam', Camera), ('f1_kps', C.c_void_p), ('f1_desc', C.c_void_p), ('f1_n', C.c_void_p), ('f1_cap', C.c_int32),
                ('f2_kps', C.c_void_p), ('f2_desc', C.c_void_p), ('f2_n', C.c_void_p), ('f2_cap', C.c_int32), ('prev_xy', C.c_void_p),
                ('window_size', C.c_int32), ('nnratio', C.c_float), ('check_orientation', C.c_int32), ('match12', C.c_void_p), ('nmatches', C.c_void_p)]


class BowBatch(C.Structure):
    _fields_ = [('kf_node', C.c_void_p), ('kf_weight', C.c_void_p), ('kf_valid', C.c_void_p), ('kf_desc', C.c_void_p), ('kf_angle', C.c_void_p), ('kf_n', C.c_void_p),
                ('kf_cap', C.c_int32), ('f_node', C.c_void_p), ('f_weight', C.c_void_p), ('f_desc', C.c_void_p), ('f_angle', C.c_void_p), ('f_n', C.c_void_p),
                ('f_cap', C.c_int32), ('f_valid', C.c_void_p), ('keyframe_pair', C.c_int32), ('nnratio', C.c_float), ('check_orientation', C.c_int32),
                ('kf_stereo', C.c_void_p), ('f_stereo', C.c_void_p), ('kf_xy', C.c_void_p), ('f_xy', C.c_void_p), ('f_octave', C.c_void_p), ('F12', C.c_void_p),
                ('epipole', C.c_void_p), ('level_sigma2', C.c_float * 16), ('scale_factors', C.c_float * 16), ('only_stereo', C.c_int32),
                ('match_f', C.c_void_p), ('nmatches', C.c_void_p)]


class FrustumBatch(C.Structure):
    _fields_ = [('cam', Camera), ('tcw', C.c_void_p), ('mp_xyz', C.c_void_p), ('mp_normal', C.c_void_p), ('mp_min_dist', C.c_void_p), ('mp_max_dist', C.c_void_p),
                ('mp_n', C.c_void_p), ('point_cap', C.c_int32), ('viewing_cos_limit', C.c_float), ('mp_inview', C.c_void_p), ('proj_x', C.c_void_p),
                ('proj_y', C.c_void_p), ('proj_xr', C.c_void_p), ('level', C.c_void_p), ('view_cos', C.c_void_p)]


class LocalMapBatch(C.Structure):
    _fields_ = [('cam', Camera),
                ('cur_kps', C.c_void_p), ('cur_desc', C.c_void_p), ('cur_uright', C.c_void_p), ('cur_n', C.c_void_p),
                ('mp_inview', C.c_void_p), ('proj_x', C.c_void_p), ('proj_y', C.c_void_p), ('proj_xr', C.c_void_p), ('level', C.c_void_p),
                ('view_cos', C.c_void_p), ('mp_desc', C.c_void_p), ('mp_obs', C.c_void_p), ('mp_n', C.c_void_p),
                ('th', C.c_float), ('nnratio', C.c_float), ('id_base', C.c_int32),
                ('f_mp', C.c_void_p), ('f_mp_obs', C.c_void_p), ('nmatches', C.c_void_p), ('ncand', C.c_void_p)]


_HEADER = os.path.join(os.path.dirname(_PKG), 'include', 'sgs_abi.h')
_BY_VALUE = {'int': C.c_int32, 'int32_t': C.c_int32, 'int64_t': C.c_int64, 'size_t': C.c_size_t, 'float': C.c_float, 'double': C.c_double}
_RETURNS = {'int': C.c_int, 'void': None}


def _ctype(decl, fn, by_value):
    """ctypes type of the C type `decl` in a prototype of `fn`: `const char*` is a byte string, every other pointer c_void_p, anything
    else must be in `by_value` (never guessed)."""
    t = ' '.join(decl.replace('*', ' * ').split()).replace(' *', '*')
    if t == 'const char*':
        return C.c_char_p
    if t.endswith('*'):
        return C.c_void_p
    t = t.removeprefix('const ')
    if t not in by_value:
        raise TypeError('%s: no ctypes mapping for the C type %r' % (fn, t))
    return by_value[t]


def parse_abi(text):
    """{name: (restype, argtypes)} of every SGS_API prototype in `text` (sgs_abi.h)."""
    text = re.sub(r'^[ \t]*#.*$', '', re.sub(r'/\*.*?\*/|//[^\n]*', ' ', text, flags=re.S), flags=re.M)
    protos = re.findall(r'SGS_API\s+([\w\s*]+?)\b(sgs_\w+)\s*\(([^)]*)\)\s*;', text)
    if len(protos) != text.count('SGS_API'):
        raise ValueError('sgs_abi.h: %d SGS_API declarations but %d prototypes parsed' % (text.count('SGS_API'), len(protos)))
    return {name: (_ctype(ret, name, _RETURNS),
                   [] if params.strip() == 'void' else [_ctype(re.sub(r'\w+\s*$', '', p), name, _BY_VALUE) for p in params.split(',')])
            for ret, name, params in protos}


with open(_HEADER) as f:
    _SIGNATURES = parse_abi(f.read())
ABI_SYMBOLS = sorted(_SIGNATURES)


def build(force=False):
    csrc = os.path.join(_PKG, 'csrc')
    if force or not os.path.exists(LIB_PATH):
        subprocess.check_call(['make', '-C', csrc, '-s', os.path.join('..', 'lib', 'libsgs_cuda.so')])
    return LIB_PATH


def lib():
    global _LIB
    if _LIB is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError('libsgs_cuda.so is not built (run __graft_entry__.build() or make -C sg-slam_b200/csrc); there is no CPU fallback')
        so = C.CDLL(LIB_PATH)
        for name, (restype, argtypes) in _SIGNATURES.items():
            fn = getattr(so, name)
            fn.restype, fn.argtypes = restype, argtypes
        _LIB = so
    return _LIB


def check(code):
    if code != SGS_OK:
        raise SgsError(code, lib().sgs_last_error().decode('utf-8', 'replace'))


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def _sized(fn, head, dtype, n_type=C.c_int, tail=()):
    """The size-query protocol of the read-out accessors: fn(*head, NULL, 0, &n, *tail) reports the element count n (SGS_ERR_CAPACITY is that
    answer, not a failure), then fn(*head, out, n, &n, *tail) fills out = zeros(n, dtype)."""
    n = n_type()
    rc = fn(*head, None, 0, C.byref(n), *tail)
    if rc != SGS_ERR_CAPACITY:
        check(rc)
    out = np.zeros(n.value, dtype)
    if n.value:
        check(fn(*head, _p(out), n.value, C.byref(n), *tail))
    return out


def device_count():
    n = C.c_int()
    check(lib().sgs_device_count(C.byref(n)))
    return n.value


class _Handle:
    """One sgs_* handle `h`: made by create(*args, &h), released once by destroy(h) on close() or garbage collection."""

    def __init__(self, create, destroy, *args):
        self.h = C.c_void_p()
        self._destroy = destroy
        check(create(*args, C.byref(self.h)))

    def close(self):
        if self.h:
            self._destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Extractor(_Handle):
    """ORB_SLAM2::ORBextractor on the GPU (sgs_extractor_* of include/sgs_abi.h)."""

    def __init__(self, width, height, nfeatures=1000, scale=1.2, nlevels=8, ini=20, mn=7, max_batch=1, device=0):
        self.params = OrbParams(nfeatures, scale, nlevels, ini, mn)
        self.width, self.height, self.max_batch, self.device = width, height, max_batch, device
        super().__init__(lib().sgs_extractor_create, lib().sgs_extractor_destroy, C.byref(self.params), width, height, max_batch, device)
        cap = C.c_int()
        check(lib().sgs_extractor_max_keypoints(self.h, C.byref(cap)))
        self.cap = cap.value

    def tables(self):
        n = self.params.nlevels
        sc, isc, s2, is2 = (np.zeros(n, np.float32) for _ in range(4))
        fpl = np.zeros(n, np.int32)
        check(lib().sgs_extractor_tables(self.h, _p(sc), _p(isc), _p(s2), _p(is2), _p(fpl)))
        return dict(scale=sc, invScale=isc, sigma2=s2, invSigma2=is2, nPerLevel=fpl)

    def level_info(self, level):
        w, h, p = C.c_int(), C.c_int(), C.c_int()
        check(lib().sgs_extractor_level_info(self.h, level, C.byref(w), C.byref(h), C.byref(p)))
        return w.value, h.value, p.value

    def extract(self, img):
        """One host image -> (keypoints [n] KP_DTYPE, descriptors [n,32] u8)."""
        img = np.ascontiguousarray(img, np.uint8)
        kps = np.zeros(self.cap, KP_DTYPE)
        desc = np.zeros((self.cap, 32), np.uint8)
        n = C.c_int()
        check(lib().sgs_extract(self.h, _p(img), img.shape[1], img.shape[0], img.strides[0], _p(kps), _p(desc), self.cap, C.byref(n)))
        return kps[:n.value].copy(), desc[:n.value].copy()

    def extract_batch(self, imgs, out_kps=None, out_desc=None, out_n=None):
        """Host batch [F,h,w] -> (kps [F,cap], desc [F,cap,32], n [F])."""
        imgs = np.ascontiguousarray(imgs, np.uint8)
        F = imgs.shape[0]
        kps = out_kps if out_kps is not None else np.zeros((F, self.cap), KP_DTYPE)
        desc = out_desc if out_desc is not None else np.zeros((F, self.cap, 32), np.uint8)
        n = out_n if out_n is not None else np.zeros(F, np.int32)
        check(lib().sgs_extract_batch(self.h, _p(imgs), F, imgs.strides[0], imgs.strides[1], _p(kps), _p(desc), self.cap, _p(n)))
        return kps, desc, n

    def extract_batch_device(self, d_ptr, nframes, frame_stride, pitch, stream=0):
        check(lib().sgs_extract_batch_device(self.h, d_ptr, nframes, frame_stride, pitch, stream))

    def fetch(self, nframes, stream=0):
        kps = np.zeros((nframes, self.cap), KP_DTYPE); desc = np.zeros((nframes, self.cap, 32), np.uint8); n = np.zeros(nframes, np.int32)
        check(lib().sgs_extractor_fetch(self.h, nframes, _p(kps), _p(desc), self.cap, _p(n), stream))
        return kps, desc, n

    def set_profiling(self, on=True):
        check(lib().sgs_extractor_set_profiling(self.h, int(on)))

    def stage_times(self):
        ms = (C.c_double * 5)(); n = C.c_int()
        check(lib().sgs_extractor_stage_times(self.h, ms, C.byref(n)))
        return [ms[i] for i in range(5)], n.value

    def results_device(self):
        k, d, c = C.c_void_p(), C.c_void_p(), C.c_void_p()
        cap = C.c_int()
        check(lib().sgs_extractor_results_device(self.h, C.byref(k), C.byref(d), C.byref(c), C.byref(cap)))
        return k.value, d.value, c.value, cap.value

    def read_level(self, frame, level, blurred=False):
        w, h, _ = self.level_info(level)
        out = np.zeros((h, w), np.uint8)
        check(lib().sgs_extractor_read_level(self.h, frame, level, int(blurred), _p(out), w))
        return out

    def read_candidates(self, frame, level):
        return _sized(lib().sgs_extractor_read_candidates, (self.h, frame, level), (np.int32, 3))


def hamming_pairs(a, b, device=0):
    a = np.ascontiguousarray(a, np.uint8); b = np.ascontiguousarray(b, np.uint8)
    out = np.zeros(len(a), np.int32)
    check(lib().sgs_hamming_pairs(_p(a), _p(b), len(a), _p(out), device))
    return out


def hamming_bf(q, t, device=0):
    q = np.ascontiguousarray(q, np.uint8); t = np.ascontiguousarray(t, np.uint8)
    bi = np.zeros(len(q), np.int32); bd = np.zeros(len(q), np.int32); sd = np.zeros(len(q), np.int32)
    check(lib().sgs_hamming_bf(_p(q), len(q), _p(t) if len(t) else None, len(t), _p(bi), _p(bd), _p(sd), device))
    return bi, bd, sd


def hamming_bf_scratch_elems(nq, nt):
    e = C.c_int64()
    check(lib().sgs_hamming_bf_scratch_elems(nq, nt, C.byref(e)))
    return e.value


def hamming_bf_device(dq, nq, dt, nt, d_idx, d_best, d_second, d_scratch=0, stream=0):
    check(lib().sgs_hamming_bf_device(dq, nq, dt, nt, d_idx, d_best, d_second, d_scratch, stream))


class HostFrame:
    """numpy arrays behind an sgs_frame_view.  bounds = (min_x, min_y, max_x, max_y) (sgs_image_bounds), default (0, 0, w, h)."""

    def __init__(self, keysUn, uRight, desc, w, h, fx, fy, cx, cy, bf, scaleFactors, bounds=None):
        self.keysUn = np.ascontiguousarray(keysUn, KP_DTYPE)
        self.uRight = np.ascontiguousarray(uRight, np.float32)
        self.desc = np.ascontiguousarray(desc, np.uint8)
        self.scaleFactors = np.ascontiguousarray(scaleFactors, np.float32)
        b = (0.0, 0.0, float(w), float(h)) if bounds is None else tuple(float(v) for v in bounds)
        self.c = FrameView(len(self.keysUn), self.keysUn.ctypes.data, self.uRight.ctypes.data, self.desc.ctypes.data,
                           *b, fx, fy, cx, cy, bf, len(self.scaleFactors), self.scaleFactors.ctypes.data)


def match_project_lastframe(cur, Tcw_cur, Tcw_last, last_has_mp, last_xyz, last_desc, last_obs, last_octave, last_angle, th,
                            mono=False, check_ori=True, cur_mp=None, cur_mp_obs=None, device=0):
    n = len(last_has_mp)
    Tc = np.ascontiguousarray(Tcw_cur, np.float32); Tl = np.ascontiguousarray(Tcw_last, np.float32)
    has = np.ascontiguousarray(last_has_mp, np.uint8); xyz = np.ascontiguousarray(last_xyz, np.float32)
    ld = np.ascontiguousarray(last_desc, np.uint8); lo = np.ascontiguousarray(last_obs, np.uint8)
    loct = np.ascontiguousarray(last_octave, np.int32); la = np.ascontiguousarray(last_angle, np.float32)
    mp = np.full(cur.c.n, -1, np.int32) if cur_mp is None else np.ascontiguousarray(cur_mp, np.int32).copy()
    mpo = None if cur_mp_obs is None else np.ascontiguousarray(cur_mp_obs, np.uint8)
    nm = C.c_int()
    check(lib().sgs_match_project_lastframe(C.byref(cur.c), _p(Tc), _p(Tl), n, _p(has), _p(xyz), _p(ld), _p(lo), _p(loct), _p(la),
                                            th, int(mono), int(check_ori), _p(mp), _p(mpo), C.byref(nm), device))
    return nm.value, mp


def match_project_keyframe(cur, Tcw_cur, kf_valid, kf_xyz, kf_desc, kf_angle, min_dist, max_dist, th, orb_dist, check_ori=True, cur_mp=None, device=0):
    """SearchByProjection(Frame&, KeyFrame*, sAlreadyFound, th, ORBdist) on the GPU: returns (nmatches, cur_mp)."""
    n = len(kf_valid)
    Tc = np.ascontiguousarray(Tcw_cur, np.float32)
    a = [np.ascontiguousarray(kf_valid, np.uint8), np.ascontiguousarray(kf_xyz, np.float32), np.ascontiguousarray(kf_desc, np.uint8),
         np.ascontiguousarray(kf_angle, np.float32), np.ascontiguousarray(min_dist, np.float32), np.ascontiguousarray(max_dist, np.float32)]
    mp = np.full(cur.c.n, -1, np.int32) if cur_mp is None else np.ascontiguousarray(cur_mp, np.int32).copy()
    nm = C.c_int()
    check(lib().sgs_match_project_keyframe(C.byref(cur.c), _p(Tc), n, *[_p(x) for x in a], th, int(orb_dist), int(check_ori), _p(mp), C.byref(nm), device))
    return nm.value, mp


def match_project_localmap(fr, inview, projx, projy, projxr, level, viewcos, mp_desc, mp_obs, th, nnratio, f_mp, f_mp_obs, id_base=0, device=0):
    n = len(inview)
    a = [np.ascontiguousarray(inview, np.uint8), np.ascontiguousarray(projx, np.float32), np.ascontiguousarray(projy, np.float32),
         np.ascontiguousarray(projxr, np.float32), np.ascontiguousarray(level, np.int32), np.ascontiguousarray(viewcos, np.float32),
         np.ascontiguousarray(mp_desc, np.uint8), np.ascontiguousarray(mp_obs, np.uint8)]
    mp = np.ascontiguousarray(f_mp, np.int32).copy(); mpo = np.ascontiguousarray(f_mp_obs, np.uint8).copy()
    nm = C.c_int()
    check(lib().sgs_match_project_localmap(C.byref(fr.c), n, *[_p(x) for x in a], th, nnratio, id_base, _p(mp), _p(mpo), C.byref(nm), device))
    return nm.value, mp, mpo


def dynreject(cur_xy, prev_xy, F, boxes, have_dyn, nfeatures, device=0):
    cur = np.ascontiguousarray(cur_xy, np.float32); prev = np.ascontiguousarray(prev_xy, np.float32)
    n = len(cur)
    Fm = None if F is None else np.ascontiguousarray(F, np.float64).reshape(9)
    bx = np.ascontiguousarray(boxes, np.float32).reshape(-1, 4) if boxes is not None and len(boxes) else np.zeros((0, 4), np.float32)
    keep = np.zeros(n, np.uint8); dist = np.zeros(n, np.float64); nk = C.c_int(); rest = C.c_int()
    check(lib().sgs_dynreject(_p(cur), _p(prev), n, _p(Fm), _p(bx) if len(bx) else None, len(bx), int(have_dyn), nfeatures, _p(keep), _p(dist),
                              C.byref(nk), C.byref(rest), device))
    return nk.value, keep, dist, bool(rest.value)


class Matcher(_Handle):
    def __init__(self, max_frames, cur_cap, point_cap, device=0):
        super().__init__(lib().sgs_matcher_create, lib().sgs_matcher_destroy, device, max_frames, cur_cap, point_cap)

    def lastframe_batch(self, args, nframes, stream=0):
        check(lib().sgs_match_project_lastframe_batch_device(self.h, C.byref(args), nframes, stream))

    def localmap_batch(self, args, nframes, stream=0):
        check(lib().sgs_match_project_localmap_batch_device(self.h, C.byref(args), nframes, stream))


def dynreject_batch_device(d_kps, d_desc, d_counts, cap, nframes, d_prev, d_F, d_boxes, d_nboxes, max_boxes, d_have, nfeatures,
                           d_kps_out, d_desc_out, d_counts_out, d_keep=0, stream=0):
    check(lib().sgs_dynreject_batch_device(d_kps, d_desc, d_counts, cap, nframes, d_prev, d_F, d_boxes, d_nboxes, max_boxes, d_have, nfeatures,
                                           d_kps_out, d_desc_out, d_counts_out, d_keep, stream))


def make_camera(w, h, cam, scale_factors, bounds=None):
    """sgs_camera with the image bounds (min_x, min_y, max_x, max_y), default (0, 0, w, h)."""
    c = Camera()
    c.min_x, c.min_y, c.max_x, c.max_y = (0.0, 0.0, float(w), float(h)) if bounds is None else tuple(float(v) for v in bounds)
    c.fx, c.fy, c.cx, c.cy, c.bf = cam['fx'], cam['fy'], cam['cx'], cam['cy'], cam['bf']
    c.nlevels = len(scale_factors)
    for i, v in enumerate(scale_factors):
        c.scale_factors[i] = float(v)
    return c


class Tracker(_Handle):
    """Batched front end with host buffers (sgs_tracker_* of include/sgs_abi.h)."""

    def __init__(self, width, height, camera, nfeatures=1000, scale=1.2, nlevels=8, ini=20, mn=7, max_batch=1, point_cap=1100, max_boxes=4, device=0):
        self.params = OrbParams(nfeatures, scale, nlevels, ini, mn)
        self.cam = camera
        super().__init__(lib().sgs_tracker_create, lib().sgs_tracker_destroy, C.byref(self.params), width, height, max_batch, point_cap, max_boxes,
                         C.byref(camera), device)
        cap = C.c_int()
        check(lib().sgs_tracker_max_keypoints(self.h, C.byref(cap)))
        self.cap, self.point_cap, self.max_boxes, self.max_batch = cap.value, point_cap, max_boxes, max_batch

    def extract(self, gray_ptr, nframes, frame_stride, pitch, kps_ptr, desc_ptr, n_ptr):
        check(lib().sgs_tracker_extract(self.h, gray_ptr, nframes, frame_stride, pitch, kps_ptr, desc_ptr, self.cap, n_ptr))

    def track(self, nframes, ptrs, th, mono, check_ori, out_ptrs):
        """ptrs: prev_xy, u_right, F, boxes, nboxes, have_dyn, last_xyz, last_desc, last_flags, last_octave, last_angle, last_n, tcw_cur, tcw_last
        out_ptrs: kps, desc, u_right (or 0), counts, cur_mp, nmatches   (all raw host addresses)"""
        check(lib().sgs_tracker_track(self.h, nframes, *ptrs, th, int(mono), int(check_ori), *out_ptrs))

    def step_rgbd_stream_device(self, det, d_rgb, rgb_stride, rgb_pitch, d_depth, depth_stride, depth_pitch, fmt, nframes, d_slot, d_new_stream, last_ptrs,
                                th, mono, check_ori, stream=0):
        """sgs_tracker_step_rgbd_stream_device: frame f is the next frame of stream slot d_slot[f]; d_new_stream: a device uint8 array or 0 (none);
        last_ptrs: the eight last-frame device arrays (xyz, desc, flags, octave, angle, n, tcw_cur, tcw_last).  Enqueued on `stream`, not synchronised."""
        check(lib().sgs_tracker_step_rgbd_stream_device(self.h, det.h, d_rgb, rgb_stride, rgb_pitch, d_depth, depth_stride, depth_pitch, C.byref(fmt), nframes,
                                                        d_slot, d_new_stream or None, *last_ptrs, th, int(mono), int(check_ori), stream or None))


class LK(_Handle):
    """cv::calcOpticalFlowPyrLK with the reference's parameters (sgs_lk_* of include/sgs_abi.h)."""
    PAD = 24            # border of every padded pyramid level (kLkPad)

    def __init__(self, width, height, max_batch=1, device=0):
        self.width, self.height = width, height
        super().__init__(lib().sgs_lk_create, lib().sgs_lk_destroy, width, height, max_batch, device)

    def track(self, cur, prev, pts):
        cur = np.ascontiguousarray(cur, np.uint8); prev = np.ascontiguousarray(prev, np.uint8)
        p = np.ascontiguousarray(pts, np.float32).reshape(-1, 2)
        out = np.zeros_like(p)
        check(lib().sgs_lk_track(self.h, _p(cur), _p(prev), cur.strides[0], _p(p), len(p), _p(out)))
        return out

    def read_level(self, which, level):
        w, h = self.width, self.height
        for _ in range(level):
            w, h = (w + 1) // 2, (h + 1) // 2
        out = np.zeros((h, w), np.uint8)
        check(lib().sgs_lk_read_level(self.h, which, level, _p(out), w))
        return out

    def read_padded(self, which, level, frame=0):
        """Padded level `level` of batch frame `frame`, border included: (image [h + 2 pad, w + 2 pad] u8, derivative plane
        dx | dy << 16 of the same shape as uint32 for which == 0, else None)."""
        w, h = self.width, self.height
        for _ in range(level):
            w, h = (w + 1) // 2, (h + 1) // 2
        p, pad = self.PAD, C.c_int()
        img = np.zeros((h + 2 * p, w + 2 * p), np.uint8)
        der = np.zeros((h + 2 * p, w + 2 * p), np.uint32) if which == 0 else None
        check(lib().sgs_lk_read_padded(self.h, which, level, frame, _p(img), _p(der), C.byref(pad)))
        assert pad.value == p, pad.value
        return img, der

    def track_batch_device(self, d_cur, d_prev, nframes, frame_stride, pitch, d_kps, d_counts, cap, d_prev_xy, stream=0, d_prev_index=0):
        """Previous images: d_prev [F], or frames of d_cur itself when d_prev_index [F] is given (then d_prev may be 0)."""
        check(lib().sgs_lk_track_batch_device(self.h, d_cur, d_prev, d_prev_index, nframes, frame_stride, pitch, d_kps, d_counts, cap, d_prev_xy, stream))


def fundamental_ransac(pts1, pts2, thresh=1.0, confidence=0.99, max_iters=1000, device=0):
    """cv::findFundamentalMat(pts1, pts2, FM_RANSAC, thresh, confidence) on the GPU.  Returns (F 3x3 or None, mask, info[4])."""
    a = np.ascontiguousarray(pts1, np.float32).reshape(-1, 2); b = np.ascontiguousarray(pts2, np.float32).reshape(-1, 2)
    F = np.zeros(9, np.float64); mask = np.zeros(len(a), np.uint8); info = np.zeros(4, np.int32)
    check(lib().sgs_fundamental_ransac(_p(a), _p(b), len(a), thresh, confidence, int(max_iters), _p(F), _p(mask), _p(info), device))
    return (None if np.isnan(F[0]) else F.reshape(3, 3)), mask, info


def fundamental_batch_device(d_kps, d_prev_xy, d_counts, cap, nframes, d_boxes, d_nboxes, d_have, max_boxes, d_prev_index, d_F, d_info,
                             thresh=1.0, confidence=0.99, max_iters=1000, stream=0):
    check(lib().sgs_fundamental_batch_device(d_kps, d_prev_xy, d_counts, cap, nframes, d_boxes, d_nboxes, d_have, max_boxes, d_prev_index,
                                             thresh, confidence, int(max_iters), d_F, d_info, stream))


def memcpy_d2h(dst_array, d_ptr):
    check(lib().sgs_memcpy_d2h(_p(dst_array), d_ptr, dst_array.nbytes))
    return dst_array


OBJ_DTYPE = np.dtype([('id', '<i4'), ('prob', '<f4'), ('x', '<f4'), ('y', '<f4'), ('w', '<f4'), ('h', '<f4')])   # sgs_object2d
DET_DIAGNOSTIC, DET_PLAN_ONLY, DET_KEEP_BLOBS = 1, 2, 4       # DET_KEEP_BLOBS: fused schedule, every materialised blob kept (a test hook)


class Detector(_Handle):
    """Detector2D (src/Detector2D.cc) on the GPU: sgs_detector_* of include/sgs_abi.h."""

    def __init__(self, param_path, bin_path, max_frames=1, det_thr=0.9, dyn_thr=0.01, flags=0, device=0):
        self.flags = flags
        super().__init__(lib().sgs_detector_create, lib().sgs_detector_destroy, os.fsencode(param_path), os.fsencode(bin_path), max_frames, det_thr,
                         dyn_thr, flags, device)
        r, t, nl, nk = C.c_int(), C.c_int(), C.c_int(), C.c_int()
        check(lib().sgs_detector_info(self.h, C.byref(r), C.byref(t), C.byref(nl), C.byref(nk)))
        self.rows_cap, self.input_size, self.num_layers, self.num_kernels = r.value, t.value, nl.value, nk.value

    def set_profiling(self, enable):
        check(lib().sgs_detector_set_profiling(self.h, int(enable)))

    def kernel_times(self):
        """(ms_total per kernel [preprocess, the kernels of describe() in order, detout_class, detout_merge], completed calls)"""
        nc = C.c_int()
        ms = _sized(lib().sgs_detector_kernel_times, (self.h,), np.float64, tail=(C.byref(nc),))
        return ms.tolist(), nc.value

    def describe(self):
        text = _sized(lib().sgs_detector_describe, (self.h,), np.uint8, C.c_int64)
        return text.tobytes().split(b'\0', 1)[0].decode()

    def detect(self, rgb):
        """One host frame (H x W x 3 uint8): accepted objects in detection order (OBJ_DTYPE)."""
        rgb = np.ascontiguousarray(rgb, np.uint8)
        out = np.zeros(self.rows_cap, OBJ_DTYPE); n = C.c_int()
        check(lib().sgs_detect(self.h, _p(rgb), rgb.shape[1], rgb.shape[0], rgb.strides[0], _p(out), len(out), C.byref(n)))
        return out[:n.value]

    def detect_device(self, d_rgb, frame_stride, pitch, width, height, nframes, d_rows=0, d_nrows=0, d_objects=0, d_nobjects=0, d_dyn_map=0,
                      d_ndyn_map=0, d_dyn_rm=0, d_ndyn_rm=0, d_have_dyn_rm=0, max_boxes=0, d_status=0, stream=0):
        check(lib().sgs_detector_detect_device(self.h, d_rgb, frame_stride, pitch, width, height, nframes, d_rows, d_nrows, d_objects, d_nobjects,
                                               d_dyn_map, d_ndyn_map, d_dyn_rm, d_ndyn_rm, d_have_dyn_rm, max_boxes, d_status, stream))

    def blob(self, name, frame=0):
        return _sized(lib().sgs_detector_blob, (self.h, name.encode(), frame), np.float32, C.c_int64)
