"""ctypes binding of libplslam_b200.so — Python mirror of the reference's operator classes.

Class and method names follow the reference (ORBextractor, LINEextractor, ORBmatcher, LSDmatcher, Optimizer);
see include/plslam_b200.h for the C ABI each method calls.
"""
import ctypes as C
import os
import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("PLSLAM_B200_LIB") or os.path.join(_HERE, "libplslam_b200.so")   # env override: A/B builds in tools/

KP_DTYPE = np.dtype([("x", "<f4"), ("y", "<f4"), ("size", "<f4"), ("angle", "<f4"),
                     ("response", "<f4"), ("octave", "<i4"), ("class_id", "<i4")])


class PLError(RuntimeError):
    pass


class PLOrbConfig(C.Structure):
    _fields_ = [("width", C.c_int), ("height", C.c_int), ("nfeatures", C.c_int), ("scale_factor", C.c_float),
                ("nlevels", C.c_int), ("ini_th_fast", C.c_int), ("min_th_fast", C.c_int), ("max_batch", C.c_int),
                ("cell_slot_cap", C.c_int)]


_lib = None
vp = C.c_void_p


def lib():
    """Load the CUDA library; there is deliberately no fallback."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise PLError(f"{LIB_PATH} is missing: run __graft_entry__.build() (no CPU fallback exists)")
        L = C.CDLL(LIB_PATH)
        L.pl_last_error.restype = C.c_char_p
        L.pl_launch_count.restype = C.c_ulonglong
        L.pl_device_bytes.restype = C.c_ulonglong
        L.pl_orb_create.argtypes = [C.POINTER(PLOrbConfig), C.POINTER(vp)]
        L.pl_orb_destroy.argtypes = [vp]
        L.pl_orb_capacity.argtypes = [vp]
        L.pl_orb_tables.argtypes = [vp] * 8
        L.pl_orb_extract.argtypes = [vp, vp, C.c_int, vp, vp, vp]
        L.pl_orb_extract_batch.argtypes = [vp, vp, C.c_int, C.c_size_t, C.c_int, vp, vp, vp]
        L.pl_orb_extract_batch_dev.argtypes = [vp, vp, C.c_int, C.c_size_t, C.c_int, vp, vp, vp, vp]
        L.pl_orb_get_level.argtypes = [vp, C.c_int, C.c_int, vp, C.c_int]
        L.pl_orb_debug_candidates.argtypes = [vp, C.c_int, C.c_int, vp, C.c_int]
        _lib = L
    return _lib


def check(rc):
    if rc < 0:
        raise PLError(f"plslam_b200 error {rc}: {lib().pl_last_error().decode()}")
    return rc


def _p(a):
    return a.ctypes.data_as(vp) if a is not None else None


def launch_count():
    return int(lib().pl_launch_count())


def device_bytes():
    """Device bytes the library's handles hold now (pl_device_bytes)."""
    return int(lib().pl_device_bytes())


class ORBextractor:
    """Mirror of ORB_SLAM2::ORBextractor (reference include/ORBextractor.h:45-111).

    `__call__(image)` == operator()(image, mask, keypoints, descriptors); the mask is ignored as in the
    reference.  `extract_batch` runs B frames per launch sequence.
    """

    def __init__(self, nfeatures, scaleFactor, nlevels, iniThFAST, minThFAST, width=640, height=480, max_batch=1,
                 cell_slot_cap=0):
        self.cfg = PLOrbConfig(width, height, nfeatures, scaleFactor, nlevels, iniThFAST, minThFAST, max_batch,
                               cell_slot_cap)
        self._h = vp()
        check(lib().pl_orb_create(C.byref(self.cfg), C.byref(self._h)))
        self.capacity = check(lib().pl_orb_capacity(self._h))
        n = nlevels
        self._scale, self._inv, self._s2, self._is2 = (np.zeros(n, np.float32) for _ in range(4))
        self.mnFeaturesPerLevel = np.zeros(n, np.int32)
        self.level_w, self.level_h = np.zeros(n, np.int32), np.zeros(n, np.int32)
        check(lib().pl_orb_tables(self._h, _p(self._scale), _p(self._inv), _p(self._s2), _p(self._is2),
                                  _p(self.mnFeaturesPerLevel), _p(self.level_w), _p(self.level_h)))

    def __del__(self):
        if getattr(self, "_h", None) and self._h.value:
            lib().pl_orb_destroy(self._h)
            self._h = vp()

    def GetLevels(self): return self.cfg.nlevels
    def GetScaleFactor(self): return self.cfg.scale_factor
    def GetScaleFactors(self): return self._scale
    def GetInverseScaleFactors(self): return self._inv
    def GetScaleSigmaSquares(self): return self._s2
    def GetInverseScaleSigmaSquares(self): return self._is2

    def __call__(self, image, mask=None):
        image = np.ascontiguousarray(image, np.uint8)
        if image.size == 0:
            return np.zeros(0, KP_DTYPE), np.zeros((0, 32), np.uint8)
        assert image.shape == (self.cfg.height, self.cfg.width)
        kps = np.zeros(self.capacity, KP_DTYPE)
        desc = np.zeros((self.capacity, 32), np.uint8)
        n = C.c_int(0)
        check(lib().pl_orb_extract(self._h, _p(image), image.strides[0], _p(kps), _p(desc), C.byref(n)))
        return kps[:n.value].copy(), desc[:n.value].copy()

    def extract_batch(self, images):
        images = np.ascontiguousarray(images, np.uint8)
        B = images.shape[0]
        kps = np.zeros((B, self.capacity), KP_DTYPE)
        desc = np.zeros((B, self.capacity, 32), np.uint8)
        n = np.zeros(B, np.int32)
        check(lib().pl_orb_extract_batch(self._h, _p(images), images.strides[1], images.strides[0], B, _p(kps),
                                         _p(desc), _p(n)))
        return kps, desc, n

    def extract_batch_dev(self, img_ptr, stride, frame_stride, B, kps_ptr, desc_ptr, n_ptr, stream=None):
        """Device-pointer variant (asynchronous)."""
        check(lib().pl_orb_extract_batch_dev(self._h, img_ptr, stride, frame_stride, B, kps_ptr, desc_ptr, n_ptr,
                                             stream))

    def mvImagePyramid(self, level, frame=0, with_border=False):
        w, h = int(self.level_w[level]), int(self.level_h[level])
        if with_border:
            w, h = w + 38, h + 38
        out = np.zeros((h, w), np.uint8)
        check(lib().pl_orb_get_level(self._h, frame, level, _p(out), int(with_border)))
        return out

    def debug_candidates(self, level, frame=0):
        n = check(lib().pl_orb_debug_candidates(self._h, frame, level, None, 0))
        out = np.zeros(max(n, 1), KP_DTYPE)
        check(lib().pl_orb_debug_candidates(self._h, frame, level, _p(out), n))
        return out[:n]


# ---------------------------------------------------------------------------------------------- matching
def _u8(a):
    return np.ascontiguousarray(a, np.uint8)


def _f32(a):
    return np.ascontiguousarray(a, np.float32)


def _i32(a):
    return np.ascontiguousarray(a, np.int32)


def frame_assign_grid(keys_un, bounds):
    """Frame::AssignFeaturesToGrid (reference src/Frame.cc:278-294) -> CSR (cell_start[3073], cell_items[n])."""
    keys = np.ascontiguousarray(keys_un); b = _f32(bounds)
    start = np.zeros(64 * 48 + 1, np.int32); items = np.zeros(max(len(keys), 1), np.int32)
    check(lib().pl_frame_assign_grid(_p(keys), len(keys), _p(b), _p(start), _p(items)))
    return start, items[:start[-1]]


class ORBmatcher:
    """Mirror of ORB_SLAM2::ORBmatcher (reference include/ORBmatcher.h:37-102) on flat frame arrays."""
    TH_HIGH, TH_LOW, HISTO_LENGTH = 100, 50, 30

    def __init__(self, nnratio=0.6, checkOri=True):
        self.mfNNratio, self.mbCheckOrientation = float(nnratio), bool(checkOri)

    @staticmethod
    def DescriptorDistance(a, b):
        a, b = _u8(a).reshape(-1, 32), _u8(b).reshape(-1, 32)
        out = np.zeros(len(a), np.int32)
        check(lib().pl_descriptor_distance_batch(_p(a), _p(b), len(a), _p(out)))
        return out if len(out) > 1 else int(out[0])

    def SearchForInitialization(self, keys1, desc1, keys2, desc2, bounds, vbPrevMatched, windowSize=10):
        k1, k2 = np.ascontiguousarray(keys1), np.ascontiguousarray(keys2)
        d1, d2 = _u8(desc1), _u8(desc2)
        pm = _f32(vbPrevMatched).copy(); b = _f32(bounds)
        m = np.zeros(max(len(k1), 1), np.int32)
        f = lib().pl_orb_search_for_initialization
        f.argtypes = [vp, vp, C.c_int, vp, vp, C.c_int, vp, vp, vp, C.c_int, C.c_float, C.c_int]
        nm = check(f(_p(k1), _p(d1), len(k1), _p(k2), _p(d2), len(k2), _p(b), _p(pm), _p(m), int(windowSize),
                     self.mfNNratio, int(self.mbCheckOrientation)))
        return nm, m[:len(k1)], pm

    def SearchByProjectionLast(self, keys_cur, desc_cur, bounds, Tcw, K, scale_factors, last_valid, last_pos,
                               last_desc, last_octave, last_angle, th, preassigned=None):
        """SearchByProjection(CurrentFrame, LastFrame, th, bMono=True)."""
        kc, dc = np.ascontiguousarray(keys_cur), _u8(desc_cur)
        arr = [_f32(bounds), _f32(Tcw), _f32(K), _f32(scale_factors), _u8(last_valid), _f32(last_pos), _u8(last_desc),
               _i32(last_octave), _f32(last_angle)]
        pre = None if preassigned is None else _u8(preassigned)
        m = np.zeros(max(len(kc), 1), np.int32)
        f = lib().pl_orb_search_by_projection_last
        f.argtypes = [vp, vp, C.c_int, vp, vp, vp, vp, C.c_int, C.c_int, vp, vp, vp, vp, vp, C.c_float, C.c_int, vp, vp]
        nm = check(f(_p(kc), _p(dc), len(kc), _p(arr[0]), _p(arr[1]), _p(arr[2]), _p(arr[3]), len(arr[3]), len(arr[4]),
                     _p(arr[4]), _p(arr[5]), _p(arr[6]), _p(arr[7]), _p(arr[8]), float(th),
                     int(self.mbCheckOrientation), _p(pre), _p(m)))
        return nm, m[:len(kc)]

    def SearchByProjectionPoints(self, keys, desc, bounds, scale_factors, in_view, proj, level, view_cos, mp_desc, th=3,
                                 preassigned=None):
        """SearchByProjection(F, vpMapPoints, th)."""
        k, d = np.ascontiguousarray(keys), _u8(desc)
        arr = [_f32(bounds), _f32(scale_factors), _u8(in_view), _f32(proj), _i32(level), _f32(view_cos), _u8(mp_desc)]
        pre = None if preassigned is None else _u8(preassigned)
        m = np.zeros(max(len(k), 1), np.int32)
        f = lib().pl_orb_search_by_projection_points
        f.argtypes = [vp, vp, C.c_int, vp, vp, C.c_int, C.c_int, vp, vp, vp, vp, vp, C.c_float, C.c_float, vp, vp]
        nm = check(f(_p(k), _p(d), len(k), _p(arr[0]), _p(arr[1]), len(arr[1]), len(arr[2]), _p(arr[2]), _p(arr[3]),
                     _p(arr[4]), _p(arr[5]), _p(arr[6]), float(th), self.mfNNratio, _p(pre), _p(m)))
        return nm, m[:len(k)]


class LSDmatcher:
    """Mirror of ORB_SLAM2::LSDmatcher (reference include/LSDmatcher.h:22-76) on flat arrays."""
    TH_HIGH, TH_LOW = 80, 50

    def __init__(self, nnratio=0.7, checkOri=True):
        self.mfNNratio, self.mbCheckOrientation = float(nnratio), bool(checkOri)

    DescriptorDistance = ORBmatcher.DescriptorDistance

    @staticmethod
    def knnMatch(d1, d2):
        """cv::BFMatcher(NORM_HAMMING).knnMatch(d1, d2, k=2) as used by FrameBFMatch."""
        d1, d2 = _u8(d1), _u8(d2)
        idx = np.zeros((max(len(d1), 1), 2), np.int32); dist = np.zeros((max(len(d1), 1), 2), np.int32)
        check(lib().pl_match_bf_knn2(_p(d1), len(d1), _p(d2), len(d2), _p(idx), _p(dist)))
        return idx[:len(d1)], dist[:len(d1)]

    def FrameBFMatch(self, ldesc1, ldesc2, TH=50.0):
        d1, d2 = _u8(ldesc1), _u8(ldesc2)
        m = np.zeros(max(len(d1), 1), np.int32)
        f = lib().pl_lsd_frame_bf_match
        f.argtypes = [vp, C.c_int, vp, C.c_int, C.c_float, C.c_float, vp]
        check(f(_p(d1), len(d1), _p(d2), len(d2), float(TH), self.mfNNratio, _p(m)))
        return m[:len(d1)]

    def SearchDouble(self, ldesc1, ldesc2):
        d1, d2 = _u8(ldesc1), _u8(ldesc2)
        m = np.zeros(max(len(d1), 1), np.int32)
        f = lib().pl_lsd_search_double
        f.argtypes = [vp, C.c_int, vp, C.c_int, C.c_float, vp]
        nm = check(f(_p(d1), len(d1), _p(d2), len(d2), self.mfNNratio, _p(m)))
        return nm, m[:len(d1)]


# ---------------------------------------------------------------------------------------------- pose-only LM
class Optimizer:
    """Mirror of ORB_SLAM2::Optimizer's pose-only entry points (reference include/Optimizer.h:56-65) on flat
    arrays: each call takes what the reference reads from the Frame and returns (n_inliers, Tcw, mvbOutlier,
    mvbLineOutlier, lm_iterations)."""

    @staticmethod
    def _run(mode, Tcw, K, pt_obs, pt_inv_sigma2, pt_Xw, line_func, line_Xw):
        Tcw, K = _f32(Tcw), _f32(K)
        po = _f32(pt_obs).reshape(-1, 2); pw = _f32(pt_inv_sigma2); px = _f32(pt_Xw).reshape(-1, 3)
        lf = np.ascontiguousarray(line_func, np.float64).reshape(-1, 3)
        lx = np.ascontiguousarray(line_Xw, np.float64).reshape(-1, 6)
        Tout = np.zeros((4, 4), np.float32)
        pout = np.zeros(max(len(po), 1), np.uint8); lout = np.zeros(max(len(lf), 1), np.uint8)
        its = C.c_int(0)
        f = lib().pl_pose_optimization
        f.argtypes = [C.c_int, vp, vp, C.c_int, vp, vp, vp, C.c_int, vp, vp, vp, vp, vp, vp]
        n = check(f(mode, _p(Tcw), _p(K), len(po), _p(po), _p(pw), _p(px), len(lf), _p(lf), _p(lx), _p(Tout), _p(pout),
                    _p(lout), C.byref(its)))
        return n, Tout, pout[:len(po)].astype(bool), lout[:len(lf)].astype(bool), its.value

    @staticmethod
    def PoseOptimization(Tcw, K, pt_obs, pt_inv_sigma2, pt_Xw, line_func, line_Xw):
        return Optimizer._run(0, Tcw, K, pt_obs, pt_inv_sigma2, pt_Xw, line_func, line_Xw)

    @staticmethod
    def PoseOptimizationWithPoints(Tcw, K, pt_obs, pt_inv_sigma2, pt_Xw):
        return Optimizer._run(1, Tcw, K, pt_obs, pt_inv_sigma2, pt_Xw, np.zeros((0, 3)), np.zeros((0, 6)))

    @staticmethod
    def PoseOptimizationWithLines(Tcw, K, line_func, line_Xw):
        return Optimizer._run(2, Tcw, K, np.zeros((0, 2)), np.zeros(0), np.zeros((0, 3)), line_func, line_Xw)


# ---------------------------------------------------------------------------------------------- line features
KEYLINE_DTYPE = np.dtype([("angle", "<f4"), ("class_id", "<i4"), ("octave", "<i4"), ("ptx", "<f4"), ("pty", "<f4"),
                          ("response", "<f4"), ("size", "<f4"), ("startPointX", "<f4"), ("startPointY", "<f4"),
                          ("endPointX", "<f4"), ("endPointY", "<f4"), ("sPointInOctaveX", "<f4"),
                          ("sPointInOctaveY", "<f4"), ("ePointInOctaveX", "<f4"), ("ePointInOctaveY", "<f4"),
                          ("lineLength", "<f4"), ("numOfPixels", "<i4")])


class PLLineConfig(C.Structure):
    _fields_ = [("width", C.c_int), ("height", C.c_int), ("nfeatures", C.c_int), ("min_line_length", C.c_double),
                ("max_batch", C.c_int), ("segment_cap", C.c_int), ("lsd_used_in_global", C.c_int)]


class LINEextractor:
    """Mirror of ORB_SLAM2::LINEextractor (reference include/LineExtractor.h:20-62).

    ctor (numOctaves, scale, nLSDFeature, min_line_length) as in the reference; `scale` reaches the detector as
    (int)scale == 1 and numOctaves is 1 in every shipped config (SURVEY.md §8a a9), which is what is implemented.
    `__call__(image, mask)` == operator()(image, mask, keylines, descriptors, lineVec2d).
    """

    def __init__(self, numOctaves=1, scale=1.2, nLSDFeature=200, min_line_length=0.0, width=640, height=480, max_batch=1,
                 segment_cap=0):
        if numOctaves != 1 or int(scale) != 1:
            raise PLError("only numOctaves == 1 and int(scale) == 1 are supported (all reference configs)")
        self.cfg = PLLineConfig(width, height, nLSDFeature, float(min_line_length), max_batch, segment_cap, 0)
        self._h = vp()
        L = lib()
        L.pl_line_create.argtypes = [C.POINTER(PLLineConfig), C.POINTER(vp)]
        L.pl_line_destroy.argtypes = [vp]
        L.pl_line_capacity.argtypes = [vp]
        L.pl_line_extract.argtypes = [vp, vp, C.c_int, vp, vp, vp, vp, vp]
        L.pl_line_extract_batch.argtypes = [vp, vp, C.c_int, C.c_size_t, C.c_int, vp, vp, vp, vp, vp]
        L.pl_line_extract_batch_dev.argtypes = [vp, vp, C.c_int, C.c_size_t, C.c_int, vp, vp, vp, vp, vp, vp]
        L.pl_line_debug_segments.argtypes = [vp, C.c_int, vp, C.c_int]
        L.pl_line_debug_scaled.argtypes = [vp, C.c_int, vp, vp, vp]
        L.pl_line_debug_sobel.argtypes = [vp, C.c_int, vp, vp]
        L.pl_line_debug_order.argtypes = [vp, C.c_int, vp, C.c_int]
        L.pl_line_debug_seed_path.argtypes = [vp]
        L.pl_line_debug_fill_order.argtypes = [vp, C.c_int]
        L.pl_line_set_undistort.argtypes = [vp, vp]
        self._und = None
        check(L.pl_line_create(C.byref(self.cfg), C.byref(self._h)))
        self.capacity = check(L.pl_line_capacity(self._h))

    def __del__(self):
        if getattr(self, "_h", None) and self._h.value:
            lib().pl_line_destroy(self._h)
            self._h = vp()

    def set_undistort(self, undistorter):
        """Take raw frames from now on and undistort them with `undistorter` (an Undistorter of the same size) inside the
        extraction, as Frame.cc:220-225 does before it calls the extractor; None takes undistorted frames again."""
        check(lib().pl_line_set_undistort(self._h, undistorter.handle if undistorter is not None else None))
        self._und = undistorter     # the map must outlive its use by this handle

    def __call__(self, image, mask=None):
        image = np.ascontiguousarray(image, np.uint8)
        if image.size == 0:
            return np.zeros(0, KEYLINE_DTYPE), np.zeros((0, 32), np.uint8), np.zeros((0, 3))
        if mask is not None and (mask.shape != image.shape or mask.dtype != np.uint8):
            raise PLError("Mask error while detecting lines: please check its dimensions and that data type is CV_8UC1")
        kl = np.zeros(self.capacity, KEYLINE_DTYPE); desc = np.zeros((self.capacity, 32), np.uint8)
        lf = np.zeros((self.capacity, 3), np.float64); n = C.c_int(0)
        m = None if mask is None else np.ascontiguousarray(mask)
        check(lib().pl_line_extract(self._h, _p(image), image.strides[0], _p(m), _p(kl), _p(desc), _p(lf), C.byref(n)))
        return kl[:n.value].copy(), desc[:n.value].copy(), lf[:n.value].copy()

    def extract_batch(self, images, mask=None):
        images = np.ascontiguousarray(images, np.uint8)
        B = images.shape[0]
        kl = np.zeros((B, self.capacity), KEYLINE_DTYPE); desc = np.zeros((B, self.capacity, 32), np.uint8)
        lf = np.zeros((B, self.capacity, 3), np.float64); n = np.zeros(B, np.int32)
        m = None if mask is None else np.ascontiguousarray(mask)
        check(lib().pl_line_extract_batch(self._h, _p(images), images.strides[1], images.strides[0], B, _p(m), _p(kl),
                                          _p(desc), _p(lf), _p(n)))
        return kl, desc, lf, n

    def extract_batch_dev(self, img_ptr, stride, frame_stride, B, mask_ptr, kl_ptr, desc_ptr, lf_ptr, n_ptr, stream=None):
        check(lib().pl_line_extract_batch_dev(self._h, img_ptr, stride, frame_stride, B, mask_ptr, kl_ptr, desc_ptr,
                                              lf_ptr, n_ptr, stream))

    # parity taps
    def debug_segments(self, frame=0):
        n = check(lib().pl_line_debug_segments(self._h, frame, None, 0))
        out = np.zeros((max(n, 1), 4), np.float32)
        check(lib().pl_line_debug_segments(self._h, frame, _p(out), n))
        return out[:n]

    def debug_scaled(self, frame=0):
        sw, sh = C.c_int(), C.c_int()
        check(lib().pl_line_debug_scaled(self._h, frame, None, C.byref(sw), C.byref(sh)))
        out = np.zeros((sh.value, sw.value), np.uint8)
        check(lib().pl_line_debug_scaled(self._h, frame, _p(out), C.byref(sw), C.byref(sh)))
        return out

    def debug_sobel(self, frame=0):
        dx = np.zeros((self.cfg.height, self.cfg.width), np.int16); dy = np.zeros_like(dx)
        check(lib().pl_line_debug_sobel(self._h, frame, _p(dx), _p(dy)))
        return dx, dy

    def debug_order(self, frame=0):
        n = check(lib().pl_line_debug_order(self._h, frame, None, 0))
        out = np.zeros(max(n, 1), np.uint32)
        check(lib().pl_line_debug_order(self._h, frame, _p(out), n))
        return out[:n]

    def debug_seed_path(self):
        """1 if the last call sorted the seeds with the cluster kernel (k_lsd_seed_order), 0 with k_lsd_hist/scan/scatter."""
        return check(lib().pl_line_debug_seed_path(self._h))

    def debug_fill_order(self, byte=0xFF):
        """Overwrite the seed order and its lengths with `byte`, so that the next call must write every entry it reports."""
        check(lib().pl_line_debug_fill_order(self._h, byte))


# ---------------------------------------------------------------------------------------------- front-end pipeline
class PLFrontendConfig(C.Structure):
    _fields_ = [("width", C.c_int), ("height", C.c_int), ("max_batch", C.c_int), ("orb_nfeatures", C.c_int),
                ("orb_scale_factor", C.c_float), ("orb_nlevels", C.c_int), ("orb_ini_th", C.c_int), ("orb_min_th", C.c_int),
                ("line_nfeatures", C.c_int), ("line_min_length", C.c_double), ("lm_cap_points", C.c_int),
                ("lm_cap_lines", C.c_int)]


class Frontend:
    """Batch front-end: ORB + LSD/LBD extraction, frame-to-frame matching, 2 x PoseOptimization per frame."""

    def __init__(self, width=640, height=480, max_batch=8, orb=(1000, 1.2, 8, 20, 7), lines=(200, 0.0), lm_caps=(512, 128)):
        self.cfg = PLFrontendConfig(width, height, max_batch, orb[0], orb[1], orb[2], orb[3], orb[4], lines[0], lines[1],
                                    lm_caps[0], lm_caps[1])
        self._h = vp()
        L = lib()
        L.pl_frontend_create.argtypes = [C.POINTER(PLFrontendConfig), C.POINTER(vp)]
        L.pl_frontend_destroy.argtypes = [vp]
        L.pl_frontend_capacities.argtypes = [vp, vp, vp]
        L.pl_frontend_set_pose_problems.argtypes = [vp, C.c_int] + [vp] * 9
        L.pl_frontend_run_dev.argtypes = [vp, vp, C.c_int, C.c_size_t, C.c_int, vp]
        L.pl_frontend_run.argtypes = [vp, vp, C.c_int, C.c_size_t, C.c_int] + [vp] * 13
        L.pl_frontend_io_bytes.argtypes = [vp, vp, vp]
        L.pl_frontend_fetch.argtypes = [vp, C.c_int] + [vp] * 12
        L.pl_frontend_set_timing.argtypes = [vp, C.c_int]
        L.pl_frontend_grow_ms.argtypes = [vp, vp]
        L.pl_frontend_grow_bytes_per_frame.argtypes = [vp]
        L.pl_frontend_grow_bytes_per_frame.restype = C.c_longlong
        L.pl_frontend_copy_poses_dev.argtypes = [vp, C.c_int, vp, vp]
        check(L.pl_frontend_create(C.byref(self.cfg), C.byref(self._h)))
        ck, cl = C.c_int(), C.c_int()
        check(L.pl_frontend_capacities(self._h, C.byref(ck), C.byref(cl)))
        self.capK, self.capL = ck.value, cl.value
        self.cap_points, self.cap_lines = lm_caps

    def __del__(self):
        if getattr(self, "_h", None) and self._h.value:
            lib().pl_frontend_destroy(self._h)
            self._h = vp()

    def set_pose_problems(self, problems):
        """problems: list of dicts from synth.synth_pose_problem (one per frame of the batch)."""
        B, cp, cl = len(problems), self.cap_points, self.cap_lines
        T0 = np.zeros((B, 16), np.float32); K = np.zeros((B, 4), np.float32)
        npt = np.zeros(B, np.int32); nln = np.zeros(B, np.int32)
        obs = np.zeros((B, cp, 2), np.float32); w = np.zeros((B, cp), np.float32); X = np.zeros((B, cp, 3), np.float32)
        lf = np.zeros((B, cl, 3), np.float64); lX = np.zeros((B, cl, 6), np.float64)
        for b, p in enumerate(problems):
            n, m = len(p["pt_obs"]), len(p["line_func"])
            assert n <= cp and m <= cl
            T0[b] = p["Tcw0"].ravel(); K[b] = p["K"]; npt[b] = n; nln[b] = m
            obs[b, :n] = p["pt_obs"]; w[b, :n] = p["pt_inv_sigma2"]; X[b, :n] = p["pt_Xw"]
            lf[b, :m] = p["line_func"]; lX[b, :m] = p["line_Xw"]
        self._problems = (T0, K, npt, obs, w, X, nln, lf, lX)
        check(lib().pl_frontend_set_pose_problems(self._h, B, _p(T0), _p(K), _p(npt), _p(obs), _p(w), _p(X), _p(nln), _p(lf), _p(lX)))

    def set_wrap(self, on=True):
        """Frame 0 is matched against the last frame of the SAME batch (closed loop) instead of the previous step's last frame."""
        lib().pl_frontend_set_wrap.argtypes = [vp, C.c_int]
        check(lib().pl_frontend_set_wrap(self._h, int(on)))

    def set_tracking(self, on=True):
        """Add the steady-state projection searches (Tracking.cc:1345-1357,1799,1855) to the step; needs pose problems (Tcw0, K)."""
        lib().pl_frontend_set_tracking.argtypes = [vp, C.c_int]
        check(lib().pl_frontend_set_tracking(self._h, int(on)))

    def fetch_tracking(self, B, which=0):
        """dict(pt_match [B][capK], n_pt, line_match [B][capL], n_line, map_pos [B][capK][3], pt_in_view, line_in_view)."""
        o = dict(pt_match=np.zeros((B, self.capK), np.int32), n_pt=np.zeros(B, np.int32), line_match=np.zeros((B, self.capL), np.int32),
                 n_line=np.zeros(B, np.int32), map_pos=np.zeros((B, self.capK, 3), np.float32), pt_in_view=np.zeros((B, self.capK), np.uint8),
                 line_in_view=np.zeros((B, self.capL), np.uint8))
        lib().pl_frontend_fetch_tracking.argtypes = [vp, C.c_int, C.c_int] + [vp] * 7
        check(lib().pl_frontend_fetch_tracking(self._h, B, which, _p(o["pt_match"]), _p(o["n_pt"]), _p(o["line_match"]), _p(o["n_line"]),
                                               _p(o["map_pos"]), _p(o["pt_in_view"]), _p(o["line_in_view"])))
        return o

    def dump(self, B, path):
        """pl_frontend_dump: the last step's results in the replay container trajectory.load_frontend reads."""
        lib().pl_frontend_dump.argtypes = [vp, C.c_int, C.c_char_p]
        check(lib().pl_frontend_dump(self._h, B, str(path).encode()))

    def pack_pose_problems(self, problems, pinned=True):
        """Pack the batch's pose problems into (pinned) host arrays for upload_pose_problems()."""
        import torch
        B, cp, cl = len(problems), self.cap_points, self.cap_lines
        shapes = [((B, 16), np.float32), ((B, 4), np.float32), ((B,), np.int32), ((B, cp, 2), np.float32), ((B, cp), np.float32),
                  ((B, cp, 3), np.float32), ((B,), np.int32), ((B, cl, 3), np.float64), ((B, cl, 6), np.float64)]
        arrs, keep = [], []
        for shp, dt in shapes:
            nbytes = int(np.prod(shp)) * np.dtype(dt).itemsize
            t = torch.zeros(max(nbytes, 1), dtype=torch.uint8, pin_memory=pinned)
            keep.append(t)
            arrs.append(t.numpy()[:nbytes].view(dt).reshape(shp))
        T0, K, npt, obs, w, X, nln, lf, lX = arrs
        for b, p in enumerate(problems):
            n, m = len(p["pt_obs"]), len(p["line_func"])
            assert n <= cp and m <= cl
            T0[b] = p["Tcw0"].ravel(); K[b] = p["K"]; npt[b] = n; nln[b] = m
            obs[b, :n] = p["pt_obs"]; w[b, :n] = p["pt_inv_sigma2"]; X[b, :n] = p["pt_Xw"]
            lf[b, :m] = p["line_func"]; lX[b, :m] = p["line_Xw"]
        self._packed = (arrs, keep, B)
        return self._packed

    def upload_pose_problems(self, stream=None):
        """Enqueue the upload of the packed problems (no synchronisation); returns the bytes enqueued."""
        arrs, _, B = self._packed
        f = lib().pl_frontend_set_pose_problems_async
        f.argtypes = [vp, C.c_int] + [vp] * 9 + [vp]
        f.restype = C.c_longlong
        return check(f(self._h, B, *[_p(a) for a in arrs], stream))

    def set_camera(self, K, distCoef):
        """mK / mDistCoef of the sequence: with k1 != 0 the step undistorts frames (for lines) and keypoints (for matching)."""
        K = _f32(K); D = _f32(distCoef)
        assert K.shape == (4,) and D.shape == (5,)
        check(lib().pl_frontend_set_camera(self._h, _p(K), _p(D)))

    def fetch_keys_un(self, B):
        out = np.zeros((B, self.capK), KP_DTYPE)
        check(lib().pl_frontend_fetch_keys_un(self._h, C.c_int(B), _p(out)))
        return out

    def alloc_outputs(self, B, pinned=False):
        shapes = dict(kps=((B, self.capK), KP_DTYPE), desc=((B, self.capK, 32), np.uint8), n=((B,), np.int32),
                      keylines=((B, self.capL), KEYLINE_DTYPE), ldesc=((B, self.capL, 32), np.uint8),
                      linefunc=((B, self.capL, 3), np.float64), nl=((B,), np.int32), pt_matches=((B, self.capK), np.int32),
                      n_pt_matches=((B,), np.int32), line_matches=((B, self.capL), np.int32), n_line_matches=((B,), np.int32),
                      poses=((2, B, 16), np.float32), inliers=((2, B), np.int32))
        out = {}
        for k, (shp, dt) in shapes.items():
            if pinned:
                import torch
                nbytes = int(np.prod(shp)) * np.dtype(dt).itemsize
                t = torch.empty(max(nbytes, 1), dtype=torch.uint8, pin_memory=True)
                out["_pin_" + k] = t
                out[k] = t.numpy()[:nbytes].view(dt).reshape(shp)
            else:
                out[k] = np.zeros(shp, dt)
        return out

    ORDER = ["kps", "desc", "n", "keylines", "ldesc", "linefunc", "nl", "pt_matches", "n_pt_matches", "line_matches",
             "n_line_matches", "poses", "inliers"]

    def run(self, images, out=None):
        """End-to-end on host buffers (images: uint8 [B][H][W])."""
        B = images.shape[0]
        out = out or self.alloc_outputs(B)
        check(lib().pl_frontend_run(self._h, _p(images), images.strides[1], images.strides[0], B,
                                    *[_p(out[k]) for k in self.ORDER]))
        return out

    def submit(self, images, out):
        """Streaming form of run(): enqueue one step (pinned host buffers); results are valid after wait()."""
        B = images.shape[0]
        check(lib().pl_frontend_submit(self._h, _p(images), C.c_int(images.strides[1]), C.c_size_t(images.strides[0]), C.c_int(B),
                                       *[_p(out[k]) for k in self.ORDER]))

    def wait(self, keep_in_flight=0):
        check(lib().pl_frontend_wait(self._h, C.c_int(keep_in_flight)))

    def run_dev(self, img_ptr, stride, frame_stride, B, stream=None):
        check(lib().pl_frontend_run_dev(self._h, img_ptr, stride, frame_stride, B, stream))

    def fetch(self, B):
        out = self.alloc_outputs(B)
        order = [k for k in self.ORDER if k != "linefunc"]
        check(lib().pl_frontend_fetch(self._h, B, *[_p(out[k]) for k in order]))
        return out

    def io_bytes(self):
        a, b = C.c_longlong(), C.c_longlong()
        check(lib().pl_frontend_io_bytes(self._h, C.byref(a), C.byref(b)))
        return a.value, b.value

    def set_timing(self, on=True):
        check(lib().pl_frontend_set_timing(self._h, int(on)))

    def grow_ms(self):
        ms = C.c_float()
        check(lib().pl_frontend_grow_ms(self._h, C.byref(ms)))
        return ms.value

    def grow_bytes_per_frame(self):
        return int(lib().pl_frontend_grow_bytes_per_frame(self._h))

    def copy_poses_dev(self, B, dst_ptr, stream=None):
        check(lib().pl_frontend_copy_poses_dev(self._h, B, dst_ptr, stream))


# ---------------------------------------------------------------------------------------------- local BA
class PLBAProblem(C.Structure):
    _fields_ = [("n_kf", C.c_int), ("kf_Tcw", vp), ("kf_fixed", vp), ("kf_K", vp), ("K_end", C.c_float * 4),
                ("n_pt", C.c_int), ("pt_Xw", vp), ("n_ln", C.c_int), ("ln_Xw", vp),
                ("n_pe", C.c_int), ("pe_kf", vp), ("pe_pt", vp), ("pe_obs", vp), ("pe_inv_sigma2", vp),
                ("n_le", C.c_int), ("le_kf", vp), ("le_ln", vp), ("le_func", vp)]


def LocalBundleAdjustmentWithLine(p, stop_flag_dev=None):
    """Optimizer::LocalBundleAdjustmentWithLine on a flattened local window (dict as made by synth.synth_ba_problem).
    Returns dict(kf_Tcw, pt_Xw, ln_Xw, pe_erase, le_erase, le_erase_kf, its)."""
    a = {k: np.ascontiguousarray(v) for k, v in p.items() if isinstance(v, np.ndarray)}
    n_kf, n_pt, n_ln, n_pe, n_le = len(a["kf_fixed"]), len(a["pt_Xw"]), len(a["ln_Xw"]), len(a["pe_kf"]), len(a["le_kf"])
    P = PLBAProblem(n_kf, _p(a["kf_Tcw"]), _p(a["kf_fixed"]), _p(a["kf_K"]), (C.c_float * 4)(*[float(v) for v in a["K_end"]]),
                    n_pt, _p(a["pt_Xw"]), n_ln, _p(a["ln_Xw"]), n_pe, _p(a["pe_kf"]), _p(a["pe_pt"]), _p(a["pe_obs"]),
                    _p(a["pe_inv_sigma2"]), n_le, _p(a["le_kf"]), _p(a["le_ln"]), _p(a["le_func"]))
    out = dict(kf_Tcw=np.zeros((n_kf, 16), np.float32), pt_Xw=np.zeros((max(n_pt, 1), 3), np.float32),
               ln_Xw=np.zeros((max(n_ln, 1), 6), np.float64), pe_erase=np.zeros(max(n_pe, 1), np.uint8),
               le_erase=np.zeros(max(n_le, 1), np.uint8), le_erase_kf=np.zeros(max(n_le, 1), np.int32))
    its = C.c_int(0)
    f = lib().pl_local_ba
    f.argtypes = [C.POINTER(PLBAProblem), vp, vp, vp, vp, vp, vp, vp, vp]
    check(f(C.byref(P), stop_flag_dev, _p(out["kf_Tcw"]), _p(out["pt_Xw"]), _p(out["ln_Xw"]), _p(out["pe_erase"]),
            _p(out["le_erase"]), _p(out["le_erase_kf"]), C.byref(its)))
    out["its"] = its.value
    for k, n in (("pt_Xw", n_pt), ("ln_Xw", n_ln), ("pe_erase", n_pe), ("le_erase", n_le), ("le_erase_kf", n_le)):
        out[k] = out[k][:n]
    return out


Optimizer.LocalBundleAdjustmentWithLine = staticmethod(LocalBundleAdjustmentWithLine)


class PLBAWindows(C.Structure):
    _fields_ = ([("W", C.c_int)] + [(f"cap_{k}", C.c_int) for k in ("kf", "pt", "ln", "pe", "le")] +
                [(f"n_{k}", vp) for k in ("kf", "pt", "ln", "pe", "le")] +
                [(k, vp) for k in ("kf_Tcw", "kf_fixed", "kf_K", "K_end", "pt_Xw", "ln_Xw", "pe_kf", "pe_pt", "pe_obs", "pe_inv_sigma2",
                                   "le_kf", "le_ln", "le_func")])


class PLBAOut(C.Structure):
    _fields_ = [(k, vp) for k in ("kf_Tcw", "pt_Xw", "ln_Xw", "pe_erase", "le_erase", "le_erase_kf", "iterations", "status")]


BA_COUNTS = ("kf", "pt", "ln", "pe", "le")
# field -> (the count its rows follow, row shape, dtype), in the [W][cap] layouts of PLBAWindows / PLBAOut
BA_INPUTS = {"kf_Tcw": ("kf", (16,), np.float32), "kf_fixed": ("kf", (), np.uint8), "kf_K": ("kf", (4,), np.float32),
             "pt_Xw": ("pt", (3,), np.float32), "ln_Xw": ("ln", (6,), np.float64), "pe_kf": ("pe", (), np.int32),
             "pe_pt": ("pe", (), np.int32), "pe_obs": ("pe", (2,), np.float32), "pe_inv_sigma2": ("pe", (), np.float32),
             "le_kf": ("le", (), np.int32), "le_ln": ("le", (), np.int32), "le_func": ("le", (3,), np.float64)}
BA_OUTPUTS = {"kf_Tcw": ("kf", (16,), np.float32), "pt_Xw": ("pt", (3,), np.float32), "ln_Xw": ("ln", (6,), np.float64),
              "pe_erase": ("pe", (), np.uint8), "le_erase": ("le", (), np.uint8), "le_erase_kf": ("le", (), np.int32)}


def _ba_lib():
    L = lib()
    if not getattr(L, "_ba_types", False):
        L.pl_local_ba_scratch_bytes.argtypes = [C.c_int] * 6
        L.pl_local_ba_scratch_bytes.restype = C.c_size_t
        L.pl_local_ba_dev.argtypes = [C.POINTER(PLBAWindows), vp, C.POINTER(PLBAOut), vp, vp]
        L._ba_types = True
    return L


def ba_window_counts(p):
    """{kf, pt, ln, pe, le} counts of one local window (dict as made by synth.synth_ba_problem)."""
    return dict(kf=len(p["kf_fixed"]), pt=len(p["pt_Xw"]), ln=len(p["ln_Xw"]), pe=len(p["pe_kf"]), le=len(p["le_kf"]))


def pack_ba_windows(problems, caps=None, fill=0):
    """Local windows (dicts as made by synth.synth_ba_problem; their sizes may differ) -> host arrays in the [W][cap] layouts of
    PLBAWindows: dict(W, caps={kf, pt, ln, pe, le}, n_kf .. n_le [W], K_end [W][4], and one [W][cap][...] array per field of
    BA_INPUTS).  caps (optional dict): capacities at least each window's counts; by default the largest count (at least 1).
    Every byte of a row past its window's count is `fill`."""
    counts = [ba_window_counts(p) for p in problems]
    W = len(problems)
    c = {k: max([1] + [n[k] for n in counts]) for k in BA_COUNTS}
    for k, v in (caps or {}).items():
        if v < c[k]:
            raise ValueError(f"cap_{k} = {v} is below a window's count {c[k]}")
        c[k] = int(v)
    out = dict(W=W, caps=c, K_end=np.array([np.asarray(p["K_end"], np.float32).reshape(4) for p in problems], np.float32).reshape(W, 4))
    for k in BA_COUNTS:
        out["n_" + k] = np.array([n[k] for n in counts], np.int32)
    for f, (k, shape, dt) in BA_INPUTS.items():
        a = np.empty((W, c[k]) + shape, dt)
        a.view(np.uint8)[...] = fill
        for w, p in enumerate(problems):
            a[w, :counts[w][k]] = np.asarray(p[f], dt).reshape((-1,) + shape)
        out[f] = a
    return out


def unpack_ba_rows(arrays, counts, fields):
    """Per-window dicts of `fields` (name -> (count, ...), as BA_INPUTS / BA_OUTPUTS) from [W][cap] arrays, each trimmed to its
    window's count: counts = {kf: [W], ...}.  Nothing past a count is read."""
    W = len(counts["kf"])
    return [{f: np.array(arrays[f][w, :int(counts[k][w])]) for f, (k, _, _) in fields.items()} for w in range(W)]


class LocalBAWindows:
    """W local windows on the device for pl_local_ba_dev (Optimizer::LocalBundleAdjustmentWithLine on each): the constructor
    packs them (pack_ba_windows) into torch CUDA tensors and allocates the outputs and the scratch once; run() only enqueues the
    launch, so it can be captured into a CUDA graph; results() waits for it and returns per-window dicts with the keys of
    LocalBundleAdjustmentWithLine plus `status`.  Output rows are pre-filled with `out_fill` bytes."""

    def __init__(self, problems, caps=None, out_fill=0):
        import torch
        h = pack_ba_windows(problems, caps)
        self.W, self.caps = h["W"], h["caps"]
        self.counts = {k: h["n_" + k] for k in BA_COUNTS}
        self.inputs = {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in h.items() if isinstance(v, np.ndarray)}
        W, c = self.W, self.caps
        self.outputs = {f: torch.empty((W, c[k]) + shape, dtype=getattr(torch, np.dtype(dt).name), device="cuda")
                        for f, (k, shape, dt) in BA_OUTPUTS.items()}
        for t in self.outputs.values():
            t.view(torch.uint8).fill_(out_fill)
        self.outputs["iterations"] = torch.full((W,), -1, dtype=torch.int32, device="cuda")
        self.outputs["status"] = torch.full((W,), -1, dtype=torch.int32, device="cuda")
        L = _ba_lib()
        caps_ = [c[k] for k in BA_COUNTS]
        self.scratch = torch.empty(max(int(L.pl_local_ba_scratch_bytes(W, *caps_)), 1), dtype=torch.uint8, device="cuda")
        ins = self.inputs
        self._win = PLBAWindows(W, *caps_, *[ins["n_" + k].data_ptr() for k in BA_COUNTS],
                                *[ins[f].data_ptr() for f in ("kf_Tcw", "kf_fixed", "kf_K", "K_end", "pt_Xw", "ln_Xw", "pe_kf",
                                                              "pe_pt", "pe_obs", "pe_inv_sigma2", "le_kf", "le_ln", "le_func")])
        self._out = PLBAOut(*[self.outputs[f].data_ptr() for f, _ in PLBAOut._fields_])
        torch.cuda.synchronize()        # the uploads ran on the current stream; run() may use another one

    def run(self, stream=None, stop_flag_dev=None):
        """pl_local_ba_dev on `stream` (a torch.cuda.Stream; None = the legacy default stream): enqueues, does not wait.
        stop_flag_dev: device address of an int32 polled like g2o's forceStopFlag, or None."""
        s = None if stream is None else stream.cuda_stream
        check(_ba_lib().pl_local_ba_dev(C.byref(self._win), stop_flag_dev, C.byref(self._out), self.scratch.data_ptr(), s))

    def results(self):
        import torch
        torch.cuda.synchronize()
        host = {k: v.cpu().numpy() for k, v in self.outputs.items()}
        res = unpack_ba_rows(host, self.counts, BA_OUTPUTS)
        for w, r in enumerate(res):
            r["its"] = int(host["iterations"][w])
            r["status"] = int(host["status"][w])
        return res



def LocalBundleAdjustmentWithLineBatch(problems, stream=None, stop_flag_dev=None):
    """Optimizer::LocalBundleAdjustmentWithLine on several windows in one pl_local_ba_dev launch (one CTA per window).
    Returns one dict per window: the keys of LocalBundleAdjustmentWithLine plus `status` (0 = ran)."""
    b = LocalBAWindows(problems)
    b.run(stream, stop_flag_dev)
    return b.results()


Optimizer.LocalBundleAdjustmentWithLineBatch = staticmethod(LocalBundleAdjustmentWithLineBatch)


def GlobalBundleAdjustemnt(p, nIterations=5, bRobust=True, stop_flag=None):
    """Optimizer::GlobalBundleAdjustemnt / BundleAdjustment with lines (Optimizer.cc:41-58,275-638; the reference's spelling) on
    a flattened map (dict as made by synth.synth_ba_problem; K_end is not read).  stop_flag: None or an int32 numpy scalar
    array the caller may set while the call runs.  Returns dict(kf_Tcw, pt_Xw, ln_Xw, its, solve_ms)."""
    a = {k: np.ascontiguousarray(v) for k, v in p.items() if isinstance(v, np.ndarray)}
    n_kf, n_pt, n_ln, n_pe, n_le = len(a["kf_fixed"]), len(a["pt_Xw"]), len(a["ln_Xw"]), len(a["pe_kf"]), len(a["le_kf"])
    P = PLBAProblem(n_kf, _p(a["kf_Tcw"]), _p(a["kf_fixed"]), _p(a["kf_K"]), (C.c_float * 4)(0, 0, 0, 0),
                    n_pt, _p(a["pt_Xw"]), n_ln, _p(a["ln_Xw"]), n_pe, _p(a["pe_kf"]), _p(a["pe_pt"]), _p(a["pe_obs"]),
                    _p(a["pe_inv_sigma2"]), n_le, _p(a["le_kf"]), _p(a["le_ln"]), _p(a["le_func"]))
    out = dict(kf_Tcw=np.zeros((n_kf, 16), np.float32), pt_Xw=np.zeros((max(n_pt, 1), 3), np.float32),
               ln_Xw=np.zeros((max(n_ln, 1), 6), np.float64))
    its = C.c_int(0); ms = C.c_float(0)
    f = lib().pl_global_ba
    f.argtypes = [C.POINTER(PLBAProblem), C.c_int, C.c_int, vp, vp, vp, vp, vp, vp]
    sf = None if stop_flag is None else _p(stop_flag)
    check(f(C.byref(P), int(nIterations), int(bool(bRobust)), sf, _p(out["kf_Tcw"]), _p(out["pt_Xw"]), _p(out["ln_Xw"]),
            C.byref(its), C.byref(ms)))
    out["its"] = its.value; out["solve_ms"] = ms.value
    out["pt_Xw"] = out["pt_Xw"][:n_pt]; out["ln_Xw"] = out["ln_Xw"][:n_ln]
    return out


Optimizer.GlobalBundleAdjustemnt = staticmethod(GlobalBundleAdjustemnt)


# ---------------------------------------------------------------------------------------------- line matching by projection
def frame_assign_grid_lines(keylines_un, bounds):
    """Frame::AssignFeaturesToGridForLine (reference src/Frame.cc:296-320) -> CSR (cell_start[3073], cell_items)."""
    kl = np.ascontiguousarray(keylines_un); b = _f32(bounds)
    cap = max(len(kl), 1) * 120
    start = np.zeros(64 * 48 + 1, np.int32); items = np.zeros(cap, np.int32)
    f = lib().pl_frame_assign_grid_lines
    f.argtypes = [vp, C.c_int, vp, vp, vp, C.c_int]
    n = check(f(_p(kl), len(kl), _p(b), _p(start), _p(items), cap))
    return start, items[:n]


def _lsd_search_last(self, keylines_cur, linefunc_cur, desc_cur, bounds, last_valid, last_proj, last_desc, last_length, th, preassigned=None):
    """LSDmatcher::SearchByProjection(CurrentFrame, LastFrame, th)."""
    kl = np.ascontiguousarray(keylines_cur)
    a = [np.ascontiguousarray(linefunc_cur, np.float64), _u8(desc_cur), _f32(bounds), _u8(last_valid), _f32(last_proj), _u8(last_desc), _f32(last_length)]
    pre = None if preassigned is None else _u8(preassigned)
    m = np.zeros(max(len(kl), 1), np.int32)
    f = lib().pl_lsd_search_by_projection_last
    f.argtypes = [vp, vp, vp, C.c_int, vp, C.c_int, vp, vp, vp, vp, C.c_float, vp, vp]
    nm = check(f(_p(kl), _p(a[0]), _p(a[1]), len(kl), _p(a[2]), len(a[3]), _p(a[3]), _p(a[4]), _p(a[5]), _p(a[6]), float(th), _p(pre), _p(m)))
    return nm, m[:len(kl)]


def _lsd_search_lines(self, keylines, linefunc, desc, bounds, in_view, proj, view_cos, ml_desc, th=3, preassigned=None):
    """LSDmatcher::SearchByProjection(F, vpMapLines, th)."""
    kl = np.ascontiguousarray(keylines)
    a = [np.ascontiguousarray(linefunc, np.float64), _u8(desc), _f32(bounds), _u8(in_view), _f32(proj), _f32(view_cos), _u8(ml_desc)]
    pre = None if preassigned is None else _u8(preassigned)
    m = np.zeros(max(len(kl), 1), np.int32)
    f = lib().pl_lsd_search_by_projection_lines
    f.argtypes = [vp, vp, vp, C.c_int, vp, C.c_int, vp, vp, vp, vp, C.c_float, C.c_float, vp, vp]
    nm = check(f(_p(kl), _p(a[0]), _p(a[1]), len(kl), _p(a[2]), len(a[3]), _p(a[3]), _p(a[4]), _p(a[5]), _p(a[6]), float(th),
                 self.mfNNratio, _p(pre), _p(m)))
    return nm, m[:len(kl)]


LSDmatcher.SearchByProjectionLast = _lsd_search_last
LSDmatcher.SearchByProjectionLines = _lsd_search_lines


# ----------------------------------------------------------------- Frame glue (reference src/Frame.cc)
class Undistorter:
    """The undistortion the mono Frame constructor does for every frame (reference src/Frame.cc:220-222:
    initUndistortRectifyMap + remap) and Frame::UndistortKeyPoints (:915-945); the map is built once per camera."""

    def __init__(self, K, distCoef, width, height):
        self.K = _f32(K); self.D = _f32(distCoef); self.w = int(width); self.h = int(height)
        assert self.K.shape == (4,) and self.D.shape == (5,)
        self.handle = vp()
        check(lib().pl_undistort_create(_p(self.K), _p(self.D), C.c_int(self.w), C.c_int(self.h), C.byref(self.handle)))

    def __del__(self):
        if getattr(self, "handle", None):
            lib().pl_undistort_destroy(self.handle); self.handle = None

    def remap(self, image):
        img = _u8(image)
        if img.shape != (self.h, self.w):
            raise PLError(f"image {img.shape} does not match the undistorter ({self.h}, {self.w})")
        out = np.empty_like(img)
        check(lib().pl_undistort_remap(self.handle, _p(img), C.c_int(self.w), _p(out), C.c_int(self.w)))
        return out

    def remap_batch_dev(self, src_ptr, sstride, sframe, B, dst_ptr, dstride, dframe, stream=None):
        check(lib().pl_undistort_remap_batch_dev(self.handle, vp(src_ptr), C.c_int(sstride), C.c_size_t(sframe), C.c_int(B),
                                                 vp(dst_ptr), C.c_int(dstride), C.c_size_t(dframe), vp(stream or 0)))

    def UndistortKeyPoints(self, keys):
        keys = np.ascontiguousarray(keys, KP_DTYPE); out = np.empty_like(keys)
        check(lib().pl_undistort_keypoints(self.handle, _p(keys), C.c_int(len(keys)), _p(out)))
        return out

    def undistort_keypoints_dev(self, kps_ptr, n_ptr, cap, B, out_ptr, stream=None):
        check(lib().pl_undistort_keypoints_dev(self.handle, vp(kps_ptr), vp(n_ptr), C.c_int(cap), C.c_int(B), vp(out_ptr),
                                               vp(stream or 0)))

    def ComputeImageBounds(self):
        return ComputeImageBounds(self.K, self.D, self.w, self.h)


def ComputeImageBounds(K, distCoef, width, height):
    """Frame::ComputeImageBounds (reference src/Frame.cc:947-985) -> [mnMinX, mnMinY, mnMaxX, mnMaxY]."""
    K = _f32(K); D = _f32(distCoef); b = np.empty(4, np.float32)
    check(lib().pl_frame_image_bounds(_p(K), _p(D), C.c_int(width), C.c_int(height), _p(b)))
    return b


def isInFrustum(Tcw, Ow, K, bounds, log_scale_factor, n_scale_levels, viewingCosLimit, pos, normal, min_dist, max_dist):
    """Frame::isInFrustum(MapPoint*, viewingCosLimit) over n map points (reference src/Frame.cc:560-620)."""
    n = len(pos)
    Tcw = _f32(Tcw); Ow = _f32(Ow); K = _f32(K); bounds = _f32(bounds)
    pos = _f32(pos); normal = _f32(normal); min_dist = _f32(min_dist); max_dist = _f32(max_dist)
    inview = np.zeros(n, np.uint8); proj = np.zeros((n, 2), np.float32); level = np.zeros(n, np.int32); vc = np.zeros(n, np.float32)
    check(lib().pl_frame_is_in_frustum_points(_p(Tcw), _p(Ow), _p(K), _p(bounds), C.c_float(log_scale_factor),
                                              C.c_int(n_scale_levels), C.c_float(viewingCosLimit), C.c_int(n), _p(pos), _p(normal),
                                              _p(min_dist), _p(max_dist), _p(inview), _p(proj), _p(level), _p(vc)))
    return inview, proj, level, vc


def isInFrustumLines(Tcw, Ow, K, bounds, log_scale_factor, viewingCosLimit, pos, normal, min_dist, max_dist):
    """Frame::isInFrustum(MapLine*, viewingCosLimit) over n map lines (reference src/Frame.cc:622-702)."""
    n = len(pos)
    Tcw = _f32(Tcw); Ow = _f32(Ow); K = _f32(K); bounds = _f32(bounds)
    pos = np.ascontiguousarray(pos, np.float64); normal = np.ascontiguousarray(normal, np.float64)
    min_dist = _f32(min_dist); max_dist = _f32(max_dist)
    inview = np.zeros(n, np.uint8); proj = np.zeros((n, 4), np.float32); level = np.zeros(n, np.int32); vc = np.zeros(n, np.float32)
    check(lib().pl_frame_is_in_frustum_lines(_p(Tcw), _p(Ow), _p(K), _p(bounds), C.c_float(log_scale_factor),
                                             C.c_float(viewingCosLimit), C.c_int(n), _p(pos), _p(normal), _p(min_dist),
                                             _p(max_dist), _p(inview), _p(proj), _p(level), _p(vc)))
    return inview, proj, level, vc


# ----------------------------------------------------------------- LocalMapping matchers (reference src/ORBmatcher.cc:720-1065)
def _fv_csr(fv):
    """DBoW2::FeatureVector (dict node -> feature indices, std::map order = ascending node id) as CSR arrays."""
    nodes = np.array(sorted(fv), np.uint32)
    start = np.zeros(len(nodes) + 1, np.int32); items = []
    for i, nd in enumerate(nodes):
        items += list(fv[int(nd)]); start[i + 1] = len(items)
    return nodes, start, np.array(items, np.int32).reshape(-1)


def _search_for_triangulation(self, keys1_un, desc1, has_mp1, keys2_un, desc2, has_mp2, fv1, fv2, F12, Cw1, R2w, t2w, K2,
                              scale_factors2, level_sigma2_2):
    """ORBmatcher::SearchForTriangulation(pKF1, pKF2, F12, vMatchedPairs, false) -> (nmatches, matches12[n1])."""
    k1 = np.ascontiguousarray(keys1_un, KP_DTYPE); k2 = np.ascontiguousarray(keys2_un, KP_DTYPE)
    d1 = _u8(desc1); d2 = _u8(desc2); m1 = _u8(has_mp1); m2 = _u8(has_mp2)
    n1a, s1, i1 = _fv_csr(fv1); n2a, s2, i2 = _fv_csr(fv2)
    F = _f32(F12); Cw = _f32(Cw1); R = _f32(R2w); t = _f32(t2w); K = _f32(K2); sf = _f32(scale_factors2); sg = _f32(level_sigma2_2)
    out = np.full(len(k1), -1, np.int32)
    nm = check(lib().pl_orb_search_for_triangulation(
        _p(k1), _p(d1), _p(m1), C.c_int(len(k1)), _p(k2), _p(d2), _p(m2), C.c_int(len(k2)), _p(n1a), _p(s1), _p(i1), C.c_int(len(n1a)),
        _p(n2a), _p(s2), _p(i2), C.c_int(len(n2a)), _p(F), _p(Cw), _p(R), _p(t), _p(K), _p(sf), _p(sg), C.c_int(len(sf)),
        C.c_int(int(self.mbCheckOrientation)), _p(out)))
    return nm, out


def _fuse_search(self, keys_un, desc, bounds, Tcw, Ow, K, scale_factors, inv_level_sigma2, log_scale_factor, skip, pos, normal,
                 min_dist, max_dist, mp_desc, th=3.0):
    """Search half of ORBmatcher::Fuse(pKF, vpMapPoints, th) -> (best_idx[n_mp], best_dist[n_mp])."""
    keys = np.ascontiguousarray(keys_un, KP_DTYPE); desc = _u8(desc)
    b = _f32(bounds); T = _f32(Tcw); O = _f32(Ow); Kc = _f32(K); sf = _f32(scale_factors); iv = _f32(inv_level_sigma2)
    n_mp = len(pos)
    sk = None if skip is None else _u8(skip)
    pos = _f32(pos); normal = _f32(normal); mn = _f32(min_dist); mx = _f32(max_dist); md = _u8(mp_desc)
    bi = np.zeros(n_mp, np.int32); bd = np.zeros(n_mp, np.int32)
    check(lib().pl_orb_fuse_search(_p(keys), _p(desc), C.c_int(len(keys)), _p(b), _p(T), _p(O), _p(Kc), _p(sf), _p(iv),
                                   C.c_int(len(sf)), C.c_float(log_scale_factor), C.c_int(n_mp), _p(sk), _p(pos), _p(normal), _p(mn),
                                   _p(mx), _p(md), C.c_float(th), _p(bi), _p(bd)))
    return bi, bd


ORBmatcher.SearchForTriangulation = _search_for_triangulation
ORBmatcher.FuseSearch = _fuse_search


def _lsd_search_for_triangulation(self, ldesc1, has_ml1, ldesc2, has_ml2, isDouble=True, th=None):
    """LSDmatcher::SearchForTriangulation(pKF1, pKF2, vMatchedPairs, isDouble) (reference src/LSDmatcher.cpp:727-776)
    -> (nmatches, vMatchedPairs[NL1]); th defaults to TH_HIGH (the 4-argument overload), th = TH_LOW + isDouble is the
    pair<> overload (:672-725)."""
    th = float(self.TH_HIGH if th is None else th)
    d1 = _u8(ldesc1).reshape(-1, 32); d2 = _u8(ldesc2).reshape(-1, 32); m1 = _u8(has_ml1); m2 = _u8(has_ml2)
    out = np.full(len(d1), -1, np.int32)
    nm = check(lib().pl_lsd_search_for_triangulation(_p(d1), _p(m1), C.c_int(len(d1)), _p(d2), _p(m2), C.c_int(len(d2)),
                                                     C.c_float(th), C.c_float(self.mfNNratio), C.c_int(int(isDouble)), _p(out)))
    return nm, out


LSDmatcher.SearchForTriangulation = _lsd_search_for_triangulation


def _search_by_bow(self, keysKF_un, descKF, has_mp_kf, keysF, descF, fvKF, fvF):
    """ORBmatcher::SearchByBoW(pKF, F, vpMapPointMatches) (reference src/ORBmatcher.cc:187-327) -> (nmatches, matchesF[F.N]):
    matchesF[j] = index of the keyframe feature whose MapPoint frame feature j receives."""
    kK = np.ascontiguousarray(keysKF_un, KP_DTYPE); kF = np.ascontiguousarray(keysF, KP_DTYPE)
    dK = _u8(descKF); dF = _u8(descF); mp = _u8(has_mp_kf)
    n1a, s1, i1 = _fv_csr(fvKF); n2a, s2, i2 = _fv_csr(fvF)
    out = np.full(len(kF), -1, np.int32)
    nm = check(lib().pl_orb_search_by_bow(_p(kK), _p(dK), _p(mp), C.c_int(len(kK)), _p(kF), _p(dF), C.c_int(len(kF)), _p(n1a), _p(s1),
                                          _p(i1), C.c_int(len(n1a)), _p(n2a), _p(s2), _p(i2), C.c_int(len(n2a)),
                                          C.c_float(self.mfNNratio), C.c_int(int(self.mbCheckOrientation)), _p(out)))
    return nm, out


ORBmatcher.SearchByBoW = _search_by_bow


def _search_by_projection_keyframe(self, keys_cur_un, desc_cur, bounds, Tcw, Ow, K, scale_factors, log_scale_factor, kf_valid, pos,
                                   mp_desc, min_dist, max_dist, kf_angle, th, ORBdist, preassigned=None):
    """ORBmatcher::SearchByProjection(CurrentFrame, pKF, sAlreadyFound, th, ORBdist) (reference src/ORBmatcher.cc:1587-1716)
    -> (nmatches, cur_match[F.N]) with cur_match[i2] = index into the keyframe's map-point list."""
    kc = np.ascontiguousarray(keys_cur_un, KP_DTYPE); dc = _u8(desc_cur)
    b = _f32(bounds); T = _f32(Tcw); O = _f32(Ow); Kc = _f32(K); sf = _f32(scale_factors)
    v = _u8(kf_valid); pos = _f32(pos); md = _u8(mp_desc); mn = _f32(min_dist); mx = _f32(max_dist); ang = _f32(kf_angle)
    pre = None if preassigned is None else _u8(preassigned)
    out = np.full(len(kc), -1, np.int32)
    nm = check(lib().pl_orb_search_by_projection_keyframe(
        _p(kc), _p(dc), C.c_int(len(kc)), _p(b), _p(T), _p(O), _p(Kc), _p(sf), C.c_int(len(sf)), C.c_float(log_scale_factor),
        C.c_int(len(v)), _p(v), _p(pos), _p(md), _p(mn), _p(mx), _p(ang), C.c_float(th), C.c_int(int(ORBdist)),
        C.c_int(int(self.mbCheckOrientation)), _p(pre), _p(out)))
    return nm, out


ORBmatcher.SearchByProjectionKeyFrame = _search_by_projection_keyframe


def _search_by_bow_keyframes(self, keys1_un, desc1, has_mp1, keys2_un, desc2, has_mp2, fv1, fv2):
    """ORBmatcher::SearchByBoW(pKF1, pKF2, vpMatches12) (reference src/ORBmatcher.cc:574-709) -> (nmatches, matches12[n1])."""
    k1 = np.ascontiguousarray(keys1_un, KP_DTYPE); k2 = np.ascontiguousarray(keys2_un, KP_DTYPE)
    d1 = _u8(desc1); d2 = _u8(desc2); m1 = _u8(has_mp1); m2 = _u8(has_mp2)
    n1a, s1, i1 = _fv_csr(fv1); n2a, s2, i2 = _fv_csr(fv2)
    out = np.full(len(k1), -1, np.int32)
    nm = check(lib().pl_orb_search_by_bow_keyframes(_p(k1), _p(d1), _p(m1), C.c_int(len(k1)), _p(k2), _p(d2), _p(m2), C.c_int(len(k2)),
                                                    _p(n1a), _p(s1), _p(i1), C.c_int(len(n1a)), _p(n2a), _p(s2), _p(i2), C.c_int(len(n2a)),
                                                    C.c_float(self.mfNNratio), C.c_int(int(self.mbCheckOrientation)), _p(out)))
    return nm, out


ORBmatcher.SearchByBoWKeyFrames = _search_by_bow_keyframes


# ---------------------------------------------------------------------------------------------- LocalMapping: map-point descriptor, line fusion
def ComputeDistinctiveDescriptors(desc, offsets, return_desc=False):
    """MapPoint::ComputeDistinctiveDescriptors (reference src/MapPoint.cc:249-314) for a batch of map points: descriptors of
    point m = rows offsets[m]..offsets[m+1] of desc.  Returns best index inside each point's list (-1 for an empty list)."""
    desc = _u8(desc).reshape(-1, 32); off = np.ascontiguousarray(offsets, np.int32)
    n = len(off) - 1
    best = np.zeros(max(n, 1), np.int32); out = np.zeros((max(n, 1), 32), np.uint8) if return_desc else None
    f = lib().pl_mappoint_distinctive_descriptors
    f.argtypes = [vp, vp, C.c_int, vp, vp]
    check(f(_p(desc), _p(off), n, _p(best), _p(out)))
    return (best[:n], out[:n]) if return_desc else best[:n]


def _lsd_fuse_search(self, keylines, kf_point_desc, bounds, Tcw, Ow, K, scale_line, log_scale_factor_line, skip, pos, normal,
                     min_dist, max_dist, ml_desc, th=3.0):
    """Search half of LSDmatcher::Fuse(pKF, vpMapLines, th) (reference src/LSDmatcher.cpp:860-1011) -> (best_idx, best_dist,
    stop_at); quirks in include/plslam_b200.h (pl_lsd_fuse_search)."""
    kl = np.ascontiguousarray(keylines); pd = _u8(kf_point_desc).reshape(-1, 32)
    b = _f32(bounds); T = _f32(Tcw); O = _f32(Ow); Kc = _f32(K)
    n = len(pos)
    sk = _u8(skip); P = np.ascontiguousarray(pos, np.float64); Nn = np.ascontiguousarray(normal, np.float64)
    mn = _f32(min_dist); mx = _f32(max_dist); md = _u8(ml_desc).reshape(-1, 32)
    bi = np.zeros(max(n, 1), np.int32); bd = np.zeros(max(n, 1), np.int32); stop = C.c_int(n)
    f = lib().pl_lsd_fuse_search
    f.argtypes = [vp, C.c_int, vp, C.c_int, vp, vp, vp, vp, C.c_float, C.c_float, C.c_int, vp, vp, vp, vp, vp, vp, C.c_float, vp, vp, vp]
    check(f(_p(kl), len(kl), _p(pd), len(pd), _p(b), _p(T), _p(O), _p(Kc), scale_line, log_scale_factor_line, n, _p(sk), _p(P), _p(Nn),
            _p(mn), _p(mx), _p(md), th, _p(bi), _p(bd), C.byref(stop)))
    return bi[:n], bd[:n], stop.value


LSDmatcher.FuseSearch = _lsd_fuse_search


# ---------------------------------------------------------------------------------------------- keyframe tables of the batched searches
def _pad_rows(arrays, dt, shape, cap, what):
    """Per-keyframe arrays -> ([n_kf][cap] + shape array of dtype dt, zero past each count; counts [n_kf]; cap).  cap defaults to
    the largest count (at least 1)."""
    counts = np.array([len(a) for a in arrays], np.int32)
    cap = max([1] + list(counts)) if cap is None else int(cap)
    if counts.size and counts.max() > cap:
        raise ValueError(f"a keyframe has {counts.max()} {what}, over the capacity {cap}")
    out = np.zeros((len(arrays), cap) + shape, dt)
    for i, a in enumerate(arrays):
        out[i, :counts[i]] = np.asarray(a, dt).reshape((-1,) + shape)
    return out, counts, cap


def _camera_rows(keyframes, **widths):
    """Per-keyframe camera fields -> float32 [n_kf][width] arrays, one per field name."""
    n_kf = len(keyframes)
    return {name: np.array([np.asarray(k[name], np.float32).reshape(w) for k in keyframes], np.float32).reshape(n_kf, w)
            for name, w in widths.items()}


def _to_device(a):
    """A host array (structured arrays as raw bytes) as a torch CUDA tensor."""
    import torch
    return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8) if a.dtype.names else np.ascontiguousarray(a)).cuda()


# ---------------------------------------------------------------------------------------------- many Fuse searches in one launch
class PLFuseProblems(C.Structure):
    _fields_ = [("P", C.c_int), ("kf", vp), ("th", vp), ("offset", vp), ("count", vp), ("out_offset", vp),
                ("n_entries", C.c_int), ("entry_lm", vp), ("entry_skip", vp), ("n_out", C.c_int)]


class PLFuseKeyframes(C.Structure):
    _fields_ = [("n_kf", C.c_int), ("cap", C.c_int), ("keys_un", vp), ("desc", vp), ("n", vp), ("Tcw", vp), ("Ow", vp), ("K", vp),
                ("bounds", vp), ("scale_factors", vp), ("inv_level_sigma2", vp), ("nlevels", C.c_int), ("log_scale_factor", C.c_float)]


class PLFuseLineKeyframes(C.Structure):
    _fields_ = [("n_kf", C.c_int), ("cap", C.c_int), ("cap_pdesc", C.c_int), ("keylines", vp), ("n", vp), ("pdesc", vp), ("n_pdesc", vp),
                ("Tcw", vp), ("Ow", vp), ("K", vp), ("bounds", vp), ("scale_line", C.c_float), ("log_scale_factor_line", C.c_float)]


class PLFuseLandmarks(C.Structure):      # PLFusePoints and PLFuseLines: the same fields, float or double positions
    _fields_ = [("n", C.c_int), ("pos", vp), ("normal", vp), ("min_dist", vp), ("max_dist", vp), ("desc", vp)]


def _fuse_lib():
    L = lib()
    if not getattr(L, "_fuse_types", False):
        L.pl_orb_fuse_search_dev.argtypes = [C.POINTER(PLFuseKeyframes), C.POINTER(PLFuseLandmarks), C.POINTER(PLFuseProblems)] + [vp] * 4
        L.pl_lsd_fuse_search_dev.argtypes = [C.POINTER(PLFuseLineKeyframes), C.POINTER(PLFuseLandmarks), C.POINTER(PLFuseProblems)] + [vp] * 5
        L._fuse_types = True
    return L


def pack_fuse_keyframes(keyframes, lines=False, cap=None, cap_pdesc=None):
    """Keyframes (dicts: keys [n] KP_DTYPE and desc [n][32] for points, kl [n] KEYLINE_DTYPE and pdesc [m][32] for lines; Tcw [16],
    Ow [3], K [4], bounds [4]) -> host arrays in the [n_kf][cap] layouts of PLFuseKeyframes / PLFuseLineKeyframes.  cap /
    cap_pdesc default to the largest count (at least 1); rows past a keyframe's count are zero."""
    cam = _camera_rows(keyframes, Tcw=16, Ow=3, K=4, bounds=4)
    rows = lambda name, dt, shape, c: _pad_rows([k[name] for k in keyframes], dt, shape, c, name)
    if lines:
        kl, n, cap = rows("kl", KEYLINE_DTYPE, (), cap)
        pdesc, n_pdesc, cap_pdesc = rows("pdesc", np.uint8, (32,), cap_pdesc)
        return dict(cam, keylines=kl, n=n, pdesc=pdesc, n_pdesc=n_pdesc, cap=cap, cap_pdesc=cap_pdesc)
    keys, n, cap = rows("keys", KP_DTYPE, (), cap)
    desc, _, _ = rows("desc", np.uint8, (32,), cap)
    return dict(cam, keys_un=keys, desc=desc, n=n, cap=cap)


def pack_fuse_problems(problems, entry_lists):
    """Problems and their entry lists -> host arrays of PLFuseProblems.  entry_lists: (lm [m] landmark rows, skip [m]) pairs, packed
    one after the other; problems: (kf, th, list) triples, `list` indexing entry_lists, so problems may share a list.  The outputs of
    problem p follow those of problem p - 1: out_offset = running sum of the counts."""
    lm = [np.asarray(l, np.int32).reshape(-1) for l, _ in entry_lists]
    sk = [np.asarray(s, np.uint8).reshape(-1) for _, s in entry_lists]
    if any(len(a) != len(b) for a, b in zip(lm, sk)):
        raise ValueError("an entry list's landmark and skip arrays differ in length")
    starts = np.cumsum([0] + [len(a) for a in lm]).astype(np.int32)
    P = len(problems)
    kf = np.array([int(p[0]) for p in problems], np.int32)
    th = np.array([float(p[1]) for p in problems], np.float32)
    offset = np.array([starts[p[2]] for p in problems], np.int32)
    count = np.array([len(lm[p[2]]) for p in problems], np.int32)
    out_offset = np.concatenate([[0], np.cumsum(count)[:-1]]).astype(np.int32) if P else np.zeros(0, np.int32)
    return dict(P=P, kf=kf, th=th, offset=offset, count=count, out_offset=out_offset,
                entry_lm=np.concatenate(lm + [np.zeros(0, np.int32)]), entry_skip=np.concatenate(sk + [np.zeros(0, np.uint8)]),
                n_out=int(count.sum()))


def pack_fuse_landmarks(landmarks, lines=False):
    """Map points or lines (dict: pos [n][3] or [n][6], normal [n][3], min_dist, max_dist [n] raw, desc [n][32]) -> host arrays."""
    ft = np.float64 if lines else np.float32
    return dict(pos=np.ascontiguousarray(landmarks["pos"], ft).reshape(-1, 6 if lines else 3),
                normal=np.ascontiguousarray(landmarks["normal"], ft).reshape(-1, 3),
                min_dist=np.ascontiguousarray(landmarks["min_dist"], np.float32).reshape(-1),
                max_dist=np.ascontiguousarray(landmarks["max_dist"], np.float32).reshape(-1),
                desc=np.ascontiguousarray(landmarks["desc"], np.uint8).reshape(-1, 32))


class FuseProblems:
    """A batch of Fuse searches on the device for pl_orb_fuse_search_dev (lines=False) or pl_lsd_fuse_search_dev (lines=True): the
    constructor packs the keyframe table, the landmark table and the problems (pack_fuse_keyframes, pack_fuse_landmarks,
    pack_fuse_problems) into torch CUDA tensors and allocates the outputs once; run() only enqueues the launch, so it can be
    captured into a CUDA graph; results() waits for it and returns one dict per problem: best_idx, best_dist (numpy, one per entry),
    status, and stop_at for lines.  scales: scale_factors, inv_level_sigma2, log_scale_factor (points) or scale_line,
    log_scale_factor_line (lines).  Outputs are pre-filled with `out_fill`."""

    def __init__(self, keyframes, landmarks, problems, entry_lists, scales, lines=False, out_fill=-7):
        import torch
        self.lines = lines
        k = pack_fuse_keyframes(keyframes, lines)
        q = pack_fuse_problems(problems, entry_lists)
        m = pack_fuse_landmarks(landmarks, lines)
        dev = _to_device
        self.host = dict(k=k, q=q, m=m)
        self.inputs = {f"k_{n}": dev(v) for n, v in k.items() if isinstance(v, np.ndarray)}
        self.inputs.update({f"q_{n}": dev(v) for n, v in q.items() if isinstance(v, np.ndarray)})
        self.inputs.update({f"m_{n}": dev(v) for n, v in m.items()})
        if not lines:
            for n in ("scale_factors", "inv_level_sigma2"):
                self.inputs[n] = dev(np.asarray(scales[n], np.float32))
        P, n_out = q["P"], q["n_out"]
        self.P, self.count = P, q["count"]
        self.outputs = {n: torch.full((max(n_out, 1),), out_fill, dtype=torch.int32, device="cuda") for n in ("best_idx", "best_dist")}
        self.outputs["status"] = torch.full((max(P, 1),), out_fill, dtype=torch.int32, device="cuda")
        if lines:
            self.outputs["stop_at"] = torch.full((max(P, 1),), out_fill, dtype=torch.int32, device="cuda")
        i = lambda n: self.inputs[n].data_ptr()
        self._q = PLFuseProblems(P, i("q_kf"), i("q_th"), i("q_offset"), i("q_count"), i("q_out_offset"), len(q["entry_lm"]),
                                 i("q_entry_lm"), i("q_entry_skip"), n_out)
        self._m = PLFuseLandmarks(len(m["desc"]), i("m_pos"), i("m_normal"), i("m_min_dist"), i("m_max_dist"), i("m_desc"))
        n_kf = len(keyframes)
        if lines:
            self._k = PLFuseLineKeyframes(n_kf, k["cap"], k["cap_pdesc"], i("k_keylines"), i("k_n"), i("k_pdesc"), i("k_n_pdesc"), i("k_Tcw"),
                                          i("k_Ow"), i("k_K"), i("k_bounds"), float(scales["scale_line"]), float(scales["log_scale_factor_line"]))
        else:
            self._k = PLFuseKeyframes(n_kf, k["cap"], i("k_keys_un"), i("k_desc"), i("k_n"), i("k_Tcw"), i("k_Ow"), i("k_K"), i("k_bounds"),
                                      i("scale_factors"), i("inv_level_sigma2"), len(scales["scale_factors"]), float(scales["log_scale_factor"]))
        torch.cuda.synchronize()        # the uploads ran on the current stream; run() may use another one

    def run(self, stream=None):
        """The launch on `stream` (a torch.cuda.Stream; None = the legacy default stream): enqueues, does not wait."""
        s = None if stream is None else stream.cuda_stream
        o = {n: t.data_ptr() for n, t in self.outputs.items()}
        L = _fuse_lib()
        if self.lines:
            check(L.pl_lsd_fuse_search_dev(C.byref(self._k), C.byref(self._m), C.byref(self._q), o["best_idx"], o["best_dist"], o["stop_at"],
                                           o["status"], s))
        else:
            check(L.pl_orb_fuse_search_dev(C.byref(self._k), C.byref(self._m), C.byref(self._q), o["best_idx"], o["best_dist"], o["status"], s))

    def results(self):
        import torch
        torch.cuda.synchronize()
        h = {n: t.cpu().numpy() for n, t in self.outputs.items()}
        q = self.host["q"]
        res = []
        for p in range(self.P):
            a, c = q["out_offset"][p], q["count"][p]
            r = dict(best_idx=h["best_idx"][a:a + c].copy(), best_dist=h["best_dist"][a:a + c].copy(), status=int(h["status"][p]))
            if self.lines:
                r["stop_at"] = int(h["stop_at"][p])
            res.append(r)
        return res


def _fuse_search_batch(self, keyframes, points, problems, entry_lists, scale_factors, inv_level_sigma2, log_scale_factor, stream=None):
    """The search half of ORBmatcher::Fuse for many (keyframe, point list) problems in one pl_orb_fuse_search_dev launch.
    keyframes, points, problems, entry_lists: see FuseProblems.  Returns one dict per problem (best_idx, best_dist, status)."""
    b = FuseProblems(keyframes, points, problems, entry_lists,
                     dict(scale_factors=scale_factors, inv_level_sigma2=inv_level_sigma2, log_scale_factor=log_scale_factor))
    b.run(stream)
    return b.results()


def _lsd_fuse_search_batch(self, keyframes, lines, problems, entry_lists, scale_line, log_scale_factor_line, stream=None):
    """The search half of LSDmatcher::Fuse for many (keyframe, line list) problems in one pl_lsd_fuse_search_dev launch.
    Returns one dict per problem (best_idx, best_dist, stop_at, status)."""
    b = FuseProblems(keyframes, lines, problems, entry_lists, dict(scale_line=scale_line, log_scale_factor_line=log_scale_factor_line),
                     lines=True)
    b.run(stream)
    return b.results()


ORBmatcher.FuseSearchBatch = _fuse_search_batch
LSDmatcher.FuseSearchBatch = _lsd_fuse_search_batch


# ---------------------------------------------------------------------------------------------- many triangulation searches in one launch
class PLTriProblems(C.Structure):
    _fields_ = [("P", C.c_int), ("kf1", vp), ("kf2", vp), ("F12", vp), ("out_offset", vp), ("n_out", C.c_int)]


class PLTriKeyframes(C.Structure):
    _fields_ = [("n_kf", C.c_int), ("cap", C.c_int), ("cap_nodes", C.c_int), ("keys_un", vp), ("desc", vp), ("has_mp", vp), ("n", vp),
                ("fv_nodes", vp), ("fv_start", vp), ("fv_items", vp), ("nn", vp), ("Tcw", vp), ("Ow", vp), ("K", vp),
                ("scale_factors", vp), ("level_sigma2", vp), ("nlevels", C.c_int)]


class PLTriLineKeyframes(C.Structure):
    _fields_ = [("n_kf", C.c_int), ("cap", C.c_int), ("ldesc", vp), ("has_ml", vp), ("n", vp)]


class PLTriLineGeometry(C.Structure):
    _fields_ = [("n_kf", C.c_int), ("cap", C.c_int), ("keylines", vp), ("line_func", vp), ("Tcw", vp), ("Ow", vp), ("K", vp),
                ("level_sigma2_line", vp), ("nlevels", C.c_int)]


class PLTriLineGroups(C.Structure):
    _fields_ = [("G", C.c_int), ("kf_cur", vp), ("entry_start", vp), ("n_entries", vp), ("out_offset", vp), ("n_entry_list", C.c_int),
                ("entry_problem", vp), ("entry_kf", vp), ("entry_median_depth", vp), ("n_out", C.c_int)]


TRI_LINE_MAX_ENTRIES = 16     # PL_TRI_LINE_MAX_ENTRIES


def _tri_lib():
    L = lib()
    if not getattr(L, "_tri_types", False):
        L.pl_orb_search_for_triangulation_dev.argtypes = [C.POINTER(PLTriKeyframes), C.POINTER(PLTriProblems), C.c_int] + [vp] * 4
        L.pl_lsd_search_for_triangulation_dev.argtypes = ([C.POINTER(PLTriLineKeyframes), C.POINTER(PLTriProblems), C.c_float, C.c_float,
                                                            C.c_int] + [vp] * 4)
        L.pl_orb_triangulate_dev.argtypes = [C.POINTER(PLTriKeyframes), C.POINTER(PLTriProblems), vp, vp, C.c_float] + [vp] * 5
        L.pl_lsd_triangulate_dev.argtypes = ([C.POINTER(PLTriLineKeyframes), C.POINTER(PLTriLineGeometry), C.POINTER(PLTriProblems)]
                                             + [vp] * 3 + [C.POINTER(PLTriLineGroups)] + [vp] * 5)
        L._tri_types = True
    return L


def pack_tri_keyframes(keyframes, lines=False, cap=None, cap_nodes=None):
    """Keyframes (dicts: keys [n] KP_DTYPE, desc [n][32], has_mp [n], fv (DBoW2 FeatureVector: dict node -> feature indices), Tcw
    [16], Ow [3], K [4] for points; ldesc [n][32], has_ml [n] for lines, and for the line triangulation keylines [n] KEYLINE_DTYPE,
    line_func [n][3], Tcw, Ow, K) -> host arrays in the [n_kf][cap] layouts of PLTriKeyframes / PLTriLineKeyframes (and
    PLTriLineGeometry when every keyframe carries keylines).  cap / cap_nodes default to the largest count (at least 1); rows past a
    keyframe's count are zero."""
    if lines:
        ldesc, n, cap = _pad_rows([k["ldesc"] for k in keyframes], np.uint8, (32,), cap, "keylines")
        has_ml, _, _ = _pad_rows([k["has_ml"] for k in keyframes], np.uint8, (), cap, "keylines")
        out = dict(ldesc=ldesc, has_ml=has_ml, n=n, cap=cap)
        if keyframes and all("keylines" in k for k in keyframes):
            out["keylines"], _, _ = _pad_rows([k["keylines"] for k in keyframes], KEYLINE_DTYPE, (), cap, "keylines")
            out["line_func"], _, _ = _pad_rows([k["line_func"] for k in keyframes], np.float64, (3,), cap, "keylines")
            out.update(_camera_rows(keyframes, Tcw=16, Ow=3, K=4))
        return out
    keys, n, cap = _pad_rows([k["keys"] for k in keyframes], KP_DTYPE, (), cap, "keypoints")
    desc, _, _ = _pad_rows([k["desc"] for k in keyframes], np.uint8, (32,), cap, "keypoints")
    has_mp, _, _ = _pad_rows([k["has_mp"] for k in keyframes], np.uint8, (), cap, "keypoints")
    csr = [_fv_csr(k["fv"]) for k in keyframes]
    nodes, nn, cap_nodes = _pad_rows([c[0] for c in csr], np.uint32, (), cap_nodes, "feature-vector nodes")
    start, _, _ = _pad_rows([c[1] for c in csr], np.int32, (), cap_nodes + 1, "feature-vector nodes")
    items, _, _ = _pad_rows([c[2] for c in csr], np.int32, (), cap, "feature-vector items")
    return dict(_camera_rows(keyframes, Tcw=16, Ow=3, K=4), keys_un=keys, desc=desc, has_mp=has_mp, n=n, fv_nodes=nodes, fv_start=start,
                fv_items=items, nn=nn, cap=cap, cap_nodes=cap_nodes)


def pack_tri_problems(problems, counts):
    """Problems (kf1, kf2) or (kf1, kf2, F12 [3][3]) -> host arrays of PLTriProblems; counts [n_kf] = the keyframes' n.  The output
    of problem p (n[kf1] entries) follows that of problem p - 1; a problem whose kf1 lies outside the table gets no output range."""
    P = len(problems)
    kf1 = np.array([int(p[0]) for p in problems], np.int32)
    kf2 = np.array([int(p[1]) for p in problems], np.int32)
    F12 = np.array([np.asarray(p[2], np.float32).reshape(9) if len(p) > 2 else np.zeros(9, np.float32) for p in problems],
                   np.float32).reshape(P, 9)
    n = np.array([counts[k] if 0 <= k < len(counts) else 0 for k in kf1], np.int32)
    out_offset = np.concatenate([[0], np.cumsum(n)[:-1]]).astype(np.int32) if P else np.zeros(0, np.int32)
    return dict(P=P, kf1=kf1, kf2=kf2, F12=F12, out_offset=out_offset, n_out=int(n.sum()), count=n)


def pack_tri_line_groups(groups, counts):
    """Line triangulation groups (dicts: kf_cur, entries = [(problem, keyframe row, median depth), ...] in TotalvMatchedIndices'
    order) -> host arrays of PLTriLineGroups; counts [n_kf] = the keyframes' n.  The groups' entries and outputs are packed end to
    end: group g owns E (E - 1) / 2 * n[kf_cur] slots after those of group g - 1 (none when kf_cur lies outside the table)."""
    G = len(groups)
    kf_cur = np.array([int(g["kf_cur"]) for g in groups], np.int32)
    n_entries = np.array([len(g["entries"]) for g in groups], np.int32)
    entry_start = np.concatenate([[0], np.cumsum(n_entries)[:-1]]).astype(np.int32) if G else np.zeros(0, np.int32)
    ent = [e for g in groups for e in g["entries"]]
    n = np.array([(counts[k] if 0 <= k < len(counts) else 0) * (E * (E - 1) // 2) for k, E in zip(kf_cur, n_entries)], np.int64)
    out_offset = np.concatenate([[0], np.cumsum(n)[:-1]]).astype(np.int32) if G else np.zeros(0, np.int32)
    return dict(G=G, kf_cur=kf_cur, entry_start=entry_start, n_entries=n_entries, out_offset=out_offset,
                entry_problem=np.array([int(e[0]) for e in ent], np.int32), entry_kf=np.array([int(e[1]) for e in ent], np.int32),
                entry_median_depth=np.array([float(e[2]) for e in ent], np.float32), n_out=int(n.sum()),
                count=n.astype(np.int32), n_cur=np.array([counts[k] if 0 <= k < len(counts) else 0 for k in kf_cur], np.int32))


class TriangulationProblems:
    """A batch of triangulation searches on the device for pl_orb_search_for_triangulation_dev (lines=False) or
    pl_lsd_search_for_triangulation_dev (lines=True): the constructor packs the keyframe table and the problems (pack_tri_keyframes,
    pack_tri_problems) into torch CUDA tensors and allocates the outputs once; run() only enqueues the launch, so it can be captured
    into a CUDA graph; results() waits for it and returns one dict per problem: matches (numpy [n[kf1]]: idx2 or -1), nmatches and
    status.  Points: scales = (scale_factors, level_sigma2), options = check_orientation; lines: options = (th, nnratio, is_double).
    Outputs are pre-filled with `out_fill` (x3D with NaN).

    Points also triangulate (LocalMapping::CreateNewMapPoints): triangulate() enqueues pl_orb_triangulate_dev on the search's device
    outputs, which it reads where run() left them, and triangulated() returns one dict per problem: code (numpy int8 [n[kf1]]: -1 no
    pair, 0 committed, 1 dropped at commit, 2 .. 8 the gate that rejected it), x3D ([n[kf1]][3], written for codes 0 and 1), nnew and
    status.

    Lines triangulate too (LocalMapping::CreateNewMapLinesConstraint) when the keyframes carry keylines, line_func, Tcw, Ow and K
    and `groups` are given (see pack_tri_line_groups; scales = level_sigma2_line): triangulate() enqueues pl_lsd_triangulate_dev and
    triangulated() returns one dict per group: code (numpy int8 [E (E - 1) / 2][n[kf_cur]], one row per entry pair in the
    reference's order, -1 .. 16 as plslam_b200.h lists them), line3D ([pairs][n[kf_cur]][6], written where the triple passed every
    gate), pairs [(i, j)], nnew and status."""

    def __init__(self, keyframes, problems, scales=None, lines=False, options=0, out_fill=-7, groups=None):
        import torch
        self.lines, self.options = lines, options
        k = pack_tri_keyframes(keyframes, lines)
        q = pack_tri_problems(problems, k["n"])
        self.host = dict(k=k, q=q)
        self.inputs = {f"k_{n}": _to_device(v) for n, v in k.items() if isinstance(v, np.ndarray)}
        self.inputs.update({f"q_{n}": _to_device(v) for n, v in q.items() if isinstance(v, np.ndarray)})
        if not lines:
            self.inputs["scale_factors"] = _to_device(np.asarray(scales[0], np.float32))
            self.inputs["level_sigma2"] = _to_device(np.asarray(scales[1], np.float32))
        self.P = q["P"]
        self.outputs = dict(matches=torch.full((max(q["n_out"], 1),), out_fill, dtype=torch.int32, device="cuda"),
                            nmatches=torch.full((max(self.P, 1),), out_fill, dtype=torch.int32, device="cuda"),
                            status=torch.full((max(self.P, 1),), out_fill, dtype=torch.int32, device="cuda"))
        if not lines:
            n_out = max(q["n_out"], 1)
            self.outputs.update(code=torch.full((n_out,), out_fill, dtype=torch.int8, device="cuda"),
                                x3D=torch.full((n_out, 3), float("nan"), dtype=torch.float32, device="cuda"),
                                nnew=torch.full((max(self.P, 1),), out_fill, dtype=torch.int32, device="cuda"),
                                tri_status=torch.full((max(self.P, 1),), out_fill, dtype=torch.int32, device="cuda"))
            self.scale_factors = np.asarray(scales[0], np.float32)
        if lines and groups is not None:
            assert scales is not None, "the line triangulation needs scales = level_sigma2_line (mvLevelSigma2Line)"
            gr = pack_tri_line_groups(groups, k["n"])
            self.host["g"] = gr
            self.inputs.update({f"g_{n}": _to_device(v) for n, v in gr.items() if isinstance(v, np.ndarray)})
            self.inputs["level_sigma2_line"] = _to_device(np.asarray(scales, np.float32).reshape(-1))
            n_out, G = max(gr["n_out"], 1), max(gr["G"], 1)
            self.outputs.update(code=torch.full((n_out,), out_fill, dtype=torch.int8, device="cuda"),
                                line3D=torch.full((n_out, 6), float("nan"), dtype=torch.float32, device="cuda"),
                                nnew=torch.full((G,), out_fill, dtype=torch.int32, device="cuda"),
                                tri_status=torch.full((G,), out_fill, dtype=torch.int32, device="cuda"))
        i = lambda n: self.inputs[n].data_ptr()
        self._q = PLTriProblems(self.P, i("q_kf1"), i("q_kf2"), None if lines else i("q_F12"), i("q_out_offset"), q["n_out"])
        n_kf = len(keyframes)
        if lines:
            self._k = PLTriLineKeyframes(n_kf, k["cap"], i("k_ldesc"), i("k_has_ml"), i("k_n"))
            if "g_kf_cur" in self.inputs:
                gr = self.host["g"]
                self._geom = PLTriLineGeometry(n_kf, k["cap"], i("k_keylines"), i("k_line_func"), i("k_Tcw"), i("k_Ow"), i("k_K"),
                                               i("level_sigma2_line"), int(self.inputs["level_sigma2_line"].numel()))
                self._g = PLTriLineGroups(gr["G"], i("g_kf_cur"), i("g_entry_start"), i("g_n_entries"), i("g_out_offset"),
                                          len(gr["entry_kf"]), i("g_entry_problem"), i("g_entry_kf"), i("g_entry_median_depth"),
                                          gr["n_out"])
        else:
            self._k = PLTriKeyframes(n_kf, k["cap"], k["cap_nodes"], i("k_keys_un"), i("k_desc"), i("k_has_mp"), i("k_n"), i("k_fv_nodes"),
                                     i("k_fv_start"), i("k_fv_items"), i("k_nn"), i("k_Tcw"), i("k_Ow"), i("k_K"), i("scale_factors"),
                                     i("level_sigma2"), len(scales[0]))
        torch.cuda.synchronize()        # the uploads ran on the current stream; run() may use another one

    def run(self, stream=None):
        """The launch on `stream` (a torch.cuda.Stream; None = the legacy default stream): enqueues, does not wait."""
        s = None if stream is None else stream.cuda_stream
        o = {n: t.data_ptr() for n, t in self.outputs.items()}
        L = _tri_lib()
        if self.lines:
            th, nnratio, is_double = self.options
            check(L.pl_lsd_search_for_triangulation_dev(C.byref(self._k), C.byref(self._q), th, nnratio, int(is_double), o["matches"],
                                                        o["nmatches"], o["status"], s))
        else:
            check(L.pl_orb_search_for_triangulation_dev(C.byref(self._k), C.byref(self._q), int(self.options), o["matches"],
                                                        o["nmatches"], o["status"], s))

    def triangulate(self, stream=None, scale_factor=None):
        """pl_orb_triangulate_dev (points) or pl_lsd_triangulate_dev (lines) on `stream` after run(): enqueues, does not wait.
        scale_factor (points): KF1's mfScaleFactor (default scale_factors[1], which a single-level table does not have)."""
        if self.lines:
            assert "g_kf_cur" in self.inputs, "the line triangulation needs groups and the keyframes' geometry"
            s = None if stream is None else stream.cuda_stream
            o = {n: t.data_ptr() for n, t in self.outputs.items()}
            check(_tri_lib().pl_lsd_triangulate_dev(C.byref(self._k), C.byref(self._geom), C.byref(self._q), o["matches"],
                                                    o["nmatches"], o["status"], C.byref(self._g), o["code"], o["line3D"], o["nnew"],
                                                    o["tri_status"], s))
            return
        if scale_factor is None:
            assert len(self.scale_factors) > 1, "nlevels == 1: pass the keyframe's mfScaleFactor"
            scale_factor = float(self.scale_factors[1])
        s = None if stream is None else stream.cuda_stream
        o = {n: t.data_ptr() for n, t in self.outputs.items()}
        check(_tri_lib().pl_orb_triangulate_dev(C.byref(self._k), C.byref(self._q), o["matches"], o["status"], float(scale_factor),
                                                o["x3D"], o["code"], o["nnew"], o["tri_status"], s))

    def triangulated(self):
        import torch
        torch.cuda.synchronize()
        h = {n: t.cpu().numpy() for n, t in self.outputs.items()}
        if self.lines:
            gr = self.host["g"]
            res = []
            for g in range(gr["G"]):
                E, n = int(gr["n_entries"][g]), int(gr["n_cur"][g])
                a, c = int(gr["out_offset"][g]), int(gr["count"][g])
                np_ = E * (E - 1) // 2
                res.append(dict(code=h["code"][a:a + c].reshape(np_, n).copy() if c else np.zeros((np_, n), np.int8),
                                line3D=h["line3D"][a:a + c].reshape(np_, n, 6).copy() if c else np.zeros((np_, n, 6), np.float32),
                                pairs=[(i, j) for i in range(E) for j in range(i + 1, E)] if np_ else [],
                                nnew=int(h["nnew"][g]), status=int(h["tri_status"][g])))
            return res
        q = self.host["q"]
        sl = lambda p: slice(q["out_offset"][p], q["out_offset"][p] + q["count"][p])
        return [dict(code=h["code"][sl(p)].copy(), x3D=h["x3D"][sl(p)].copy(), nnew=int(h["nnew"][p]), status=int(h["tri_status"][p]))
                for p in range(self.P)]

    def results(self):
        import torch
        torch.cuda.synchronize()
        h = {n: t.cpu().numpy() for n, t in self.outputs.items()}
        q = self.host["q"]
        return [dict(matches=h["matches"][q["out_offset"][p]:q["out_offset"][p] + q["count"][p]].copy(),
                     nmatches=int(h["nmatches"][p]), status=int(h["status"][p])) for p in range(self.P)]


def _search_for_triangulation_batch(self, keyframes, problems, scale_factors, level_sigma2, stream=None):
    """ORBmatcher::SearchForTriangulation for many (KF1, KF2, F12) problems in one pl_orb_search_for_triangulation_dev launch.
    keyframes, problems: see TriangulationProblems.  Returns one dict per problem (matches, nmatches, status)."""
    b = TriangulationProblems(keyframes, problems, (scale_factors, level_sigma2), options=int(self.mbCheckOrientation))
    b.run(stream)
    return b.results()


def _lsd_search_for_triangulation_batch(self, keyframes, problems, isDouble=True, th=None, stream=None):
    """LSDmatcher::SearchForTriangulation for many (KF1, KF2) problems in one pl_lsd_search_for_triangulation_dev launch; th defaults
    to TH_HIGH as in SearchForTriangulation.  Returns one dict per problem (matches, nmatches, status)."""
    b = TriangulationProblems(keyframes, problems, lines=True,
                              options=(float(self.TH_HIGH if th is None else th), float(self.mfNNratio), bool(isDouble)))
    b.run(stream)
    return b.results()


ORBmatcher.SearchForTriangulationBatch = _search_for_triangulation_batch
LSDmatcher.SearchForTriangulationBatch = _lsd_search_for_triangulation_batch


# ---------------------------------------------------------------------------------------------- redundant keyframes (KeyFrameCulling)
class PLCullKeyframes(C.Structure):
    _fields_ = [("n_kf", C.c_int), ("cap", C.c_int), ("keys_un", vp), ("n", vp), ("mp", vp), ("origin", vp), ("not_erase", vp)]


class PLCullPoints(C.Structure):
    _fields_ = [("n_mp", C.c_int), ("n_obs", C.c_int), ("bad", vp), ("obs_offset", vp), ("obs_kf", vp), ("obs_idx", vp)]


class PLCullGroups(C.Structure):
    _fields_ = [("G", C.c_int), ("offset", vp), ("count", vp), ("n_list", C.c_int), ("list", vp)]


def _cull_lib():
    L = lib()
    if not getattr(L, "_cull_types", False):
        L.pl_keyframe_culling_dev.argtypes = [C.POINTER(PLCullKeyframes), C.POINTER(PLCullPoints), C.POINTER(PLCullGroups)] + [vp] * 5
        L._cull_types = True
    return L


def pack_cull_keyframes(keyframes, cap=None):
    """Keyframes (dicts: keys [n] KP_DTYPE (mvKeysUn; the octave is read), mp [n] (GetMapPointMatches(): map-point index or -1),
    origin (mnId == 0), not_erase (mbNotErase)) -> host arrays in the [n_kf][cap] layout of PLCullKeyframes.  cap defaults to the
    largest count (at least 1); slots past a keyframe's count are -1."""
    keys, n, cap = _pad_rows([k["keys"] for k in keyframes], KP_DTYPE, (), cap, "keypoints")
    mp, _, _ = _pad_rows([np.asarray(k["mp"], np.int32) + 1 for k in keyframes], np.int32, (), cap, "keypoints")
    return dict(keys_un=keys, n=n, mp=mp - 1, origin=np.array([bool(k["origin"]) for k in keyframes], np.uint8),
                not_erase=np.array([bool(k["not_erase"]) for k in keyframes], np.uint8), cap=cap)


def pack_cull_points(points):
    """Map points (dict: bad [n_mp], observations = per point the (keyframe row, idx) pairs of GetObservations(), in any order) ->
    host arrays of PLCullPoints (the observations as CSR)."""
    obs = points["observations"]
    offset = np.zeros(len(obs) + 1, np.int32)
    offset[1:] = np.cumsum([len(o) for o in obs])
    flat = np.array([e for o in obs for e in o], np.int32).reshape(-1, 2)
    return dict(bad=np.asarray(points["bad"], np.uint8).reshape(-1), obs_offset=offset, obs_kf=flat[:, 0].copy(),
                obs_idx=flat[:, 1].copy())


def pack_cull_groups(groups):
    """Groups (one list of keyframe rows per current keyframe, GetVectorCovisibleKeyFrames() order) -> host arrays of PLCullGroups,
    the lists packed end to end."""
    count = np.array([len(g) for g in groups], np.int32)
    offset = np.concatenate([[0], np.cumsum(count)[:-1]]).astype(np.int32) if len(groups) else np.zeros(0, np.int32)
    return dict(offset=offset, count=count, list=np.array([int(k) for g in groups for k in g], np.int32))


class KeyFrameCullingProblems:
    """A batch of KeyFrameCulling groups on the device for pl_keyframe_culling_dev: the constructor takes the packed host arrays
    (pack_cull_keyframes, pack_cull_points, pack_cull_groups; one dict each, any of their arrays may be replaced), uploads them as
    torch CUDA tensors and allocates the outputs once; run() only enqueues the launch, so it can be captured into a CUDA graph;
    results() waits for it and returns one dict per group: code (numpy int8, one per list entry: -1 skipped, 0 kept, 1 culled,
    2 redundant but mbNotErase), n_mps, n_redundant (numpy int32, per entry) and status.  Outputs are pre-filled with `out_fill`."""

    def __init__(self, keyframes, points, groups, out_fill=-7):
        import torch
        self.host = dict(k=keyframes, m=points, g=groups)
        self.inputs = {f"k_{n}": _to_device(keyframes[n]) for n in ("keys_un", "n", "mp", "origin", "not_erase")}
        self.inputs.update({f"m_{n}": _to_device(points[n]) for n in ("bad", "obs_offset", "obs_kf", "obs_idx")})
        self.inputs.update({f"g_{n}": _to_device(groups[n]) for n in ("offset", "count", "list")})
        self.G, n_list = len(groups["offset"]), len(groups["list"])
        self.outputs = dict(code=torch.full((max(n_list, 1),), out_fill, dtype=torch.int8, device="cuda"),
                            n_mps=torch.full((max(n_list, 1),), out_fill, dtype=torch.int32, device="cuda"),
                            n_redundant=torch.full((max(n_list, 1),), out_fill, dtype=torch.int32, device="cuda"),
                            status=torch.full((max(self.G, 1),), out_fill, dtype=torch.int32, device="cuda"))
        i = lambda n: self.inputs[n].data_ptr()
        self._k = PLCullKeyframes(len(keyframes["n"]), int(keyframes["mp"].shape[1]), i("k_keys_un"), i("k_n"), i("k_mp"), i("k_origin"),
                                  i("k_not_erase"))
        self._m = PLCullPoints(len(points["bad"]), len(points["obs_kf"]), i("m_bad"), i("m_obs_offset"), i("m_obs_kf"), i("m_obs_idx"))
        self._g = PLCullGroups(self.G, i("g_offset"), i("g_count"), n_list, i("g_list"))
        torch.cuda.synchronize()        # the uploads ran on the current stream; run() may use another one

    def run(self, stream=None):
        """The launch on `stream` (a torch.cuda.Stream; None = the legacy default stream): enqueues, does not wait."""
        s = None if stream is None else stream.cuda_stream
        o = {n: t.data_ptr() for n, t in self.outputs.items()}
        check(_cull_lib().pl_keyframe_culling_dev(C.byref(self._k), C.byref(self._m), C.byref(self._g), o["code"], o["n_mps"],
                                                  o["n_redundant"], o["status"], s))

    def results(self):
        import torch
        torch.cuda.synchronize()
        h = {n: t.cpu().numpy() for n, t in self.outputs.items()}
        g = self.host["g"]
        out = []
        for q in range(self.G):
            a, c = int(g["offset"][q]), int(g["count"][q])
            sl = slice(a, a + c) if a >= 0 and c >= 0 else slice(0, 0)
            out.append(dict(code=h["code"][sl].copy(), n_mps=h["n_mps"][sl].copy(), n_redundant=h["n_redundant"][sl].copy(),
                            status=int(h["status"][q])))
        return out


def KeyFrameCullingBatch(keyframes, points, groups, stream=None):
    """LocalMapping::KeyFrameCulling for many current keyframes in one pl_keyframe_culling_dev launch: keyframes, points and groups
    as pack_cull_keyframes, pack_cull_points and pack_cull_groups take them.  Returns one dict per group (code, n_mps, n_redundant,
    status); the caller calls SetBadFlag() on the entries with codes 1 and 2, in list order."""
    b = KeyFrameCullingProblems(pack_cull_keyframes(keyframes), pack_cull_points(points), pack_cull_groups(groups))
    b.run(stream)
    return b.results()


# ---------------------------------------------------------------------------------------------- tracking against a fixed map
class PLMapDesc(C.Structure):
    _fields_ = [("n_points", C.c_int), ("pt_pos", vp), ("pt_normal", vp), ("pt_min_dist", vp), ("pt_max_dist", vp), ("pt_desc", vp),
                ("n_lines", C.c_int), ("ln_pos", vp), ("ln_normal", vp), ("ln_min_dist", vp), ("ln_max_dist", vp), ("ln_desc", vp)]


class PLTrackFrames(C.Structure):
    _fields_ = [("B", C.c_int), ("keys_un", vp), ("desc", vp), ("n", vp), ("cap_points", C.c_int), ("keylines", vp), ("line_func", vp),
                ("line_desc", vp), ("nl", vp), ("cap_lines", C.c_int), ("bounds", vp), ("scale_factors", vp), ("inv_level_sigma2", vp),
                ("nlevels", C.c_int), ("log_scale_factor", C.c_float), ("Tcw0", vp), ("K", vp), ("point_map_in", vp), ("line_map_in", vp)]


class PLTrackLocal(C.Structure):
    _fields_ = [("pt_offset", vp), ("pt_count", vp), ("pt_index", vp), ("n_pt_index", C.c_int), ("cap_local_points", C.c_int),
                ("ln_offset", vp), ("ln_count", vp), ("ln_index", vp), ("n_ln_index", C.c_int), ("cap_local_lines", C.c_int),
                ("frames_since_reloc", vp), ("max_frames", C.c_int)]


_TRACK_OUT = ["Tcw", "point_map", "point_outlier", "line_map", "line_outlier", "inliers", "ok", "pt_in_view", "pt_proj", "pt_level",
              "pt_view_cos", "ln_in_view", "ln_proj", "ln_level", "ln_view_cos", "pt_match", "ln_match", "prob_n_points", "prob_pt_obs",
              "prob_pt_inv_sigma2", "prob_pt_Xw", "prob_n_lines", "prob_line_func", "prob_line_Xw"]
_TAPS = _TRACK_OUT[7:]


class PLTrackOut(C.Structure):
    _fields_ = [(k, vp) for k in _TRACK_OUT]


def _track_lib():
    L = lib()
    if not getattr(L, "_track_types", False):
        L.pl_map_create.argtypes = [C.POINTER(PLMapDesc), C.POINTER(vp)]
        L.pl_map_destroy.argtypes = [vp]
        L.pl_map_check_indices.argtypes = [vp]
        L.pl_track_local_map_scratch_bytes.argtypes = [C.c_int] * 5
        L.pl_track_local_map_scratch_bytes.restype = C.c_size_t
        L.pl_track_local_map_dev.argtypes = [vp, C.POINTER(PLTrackFrames), C.POINTER(PLTrackLocal), C.POINTER(PLTrackOut), vp, vp]
        L.pl_track_local_map.argtypes = [vp, C.POINTER(PLTrackFrames), C.POINTER(PLTrackLocal), C.POINTER(PLTrackOut)]
        L.pl_frontend_track_local_map_dev.argtypes = [vp, vp, C.c_int, vp, vp, vp, vp, C.POINTER(PLTrackLocal), C.POINTER(PLTrackOut), vp, vp]
        L.pl_track_local_map_seen_dev.argtypes = [vp, C.POINTER(PLTrackFrames), vp, vp, C.POINTER(PLTrackLocal), C.POINTER(PLTrackOut), vp, vp]
        L.pl_track_motion_model_scratch_bytes.argtypes = [C.c_int] * 3
        L.pl_track_motion_model_scratch_bytes.restype = C.c_size_t
        L.pl_track_motion_model_dev.argtypes = [vp, C.POINTER(PLTrackFrames), C.POINTER(PLTrackLast), C.POINTER(PLTrackMotionOut), vp, vp]
        L.pl_track_motion_model.argtypes = [vp, C.POINTER(PLTrackFrames), C.POINTER(PLTrackLast), C.POINTER(PLTrackMotionOut)]
        L.pl_track_velocity_dev.argtypes = [C.c_int, vp, vp, vp, vp, vp]
        L.pl_map_set_keyframes.argtypes = [vp, C.POINTER(PLKeyFrameGraphDesc)]
        L.pl_map_check_capacity.argtypes = [vp]
        L.pl_track_update_local_map_dev.argtypes = [vp, C.c_int, vp, C.c_int, vp, vp, C.POINTER(PLLocalMap), vp]
        L.pl_track_local_map_lists_scratch_bytes.argtypes = [C.c_int] * 5
        L.pl_track_local_map_lists_scratch_bytes.restype = C.c_size_t
        L.pl_track_local_map_lists_dev.argtypes = [vp, C.POINTER(PLTrackFrames), vp, vp, C.POINTER(PLLocalMap), vp, C.c_int, vp, vp,
                                                   C.POINTER(PLTrackOut), vp, vp]
        L.pl_track_relative_pose_dev.argtypes = [vp, C.c_int, vp, vp, vp, vp]
        L.pl_track_last_pose_dev.argtypes = [vp, C.c_int, vp, vp, vp, vp]
        L._track_types = True
    return L


class Map:
    """A fixed map on the device (pl_map_create): map points (GetWorldPos, GetNormal, raw mfMinDistance / mfMaxDistance,
    GetDescriptor) and map lines (mWorldPos, GetNormal, raw distances, GetDescriptor), indexed 0..n-1."""

    def __init__(self, pt_pos, pt_normal, pt_min_dist, pt_max_dist, pt_desc, ln_pos, ln_normal, ln_min_dist, ln_max_dist, ln_desc):
        self._a = [_f32(pt_pos).reshape(-1, 3), _f32(pt_normal).reshape(-1, 3), _f32(pt_min_dist), _f32(pt_max_dist),
                   np.ascontiguousarray(pt_desc, np.uint8).reshape(-1, 32), np.ascontiguousarray(ln_pos, np.float64).reshape(-1, 6),
                   np.ascontiguousarray(ln_normal, np.float64).reshape(-1, 3), _f32(ln_min_dist), _f32(ln_max_dist),
                   np.ascontiguousarray(ln_desc, np.uint8).reshape(-1, 32)]
        a = self._a
        self.n_points, self.n_lines = len(a[0]), len(a[5])
        d = PLMapDesc(self.n_points, *[_p(x) for x in a[:5]], self.n_lines, *[_p(x) for x in a[5:]])
        self._h = vp()
        check(_track_lib().pl_map_create(C.byref(d), C.byref(self._h)))

    def __del__(self):
        if getattr(self, "_h", None) and self._h.value:
            lib().pl_map_destroy(self._h)
            self._h = vp()

    def check_indices(self):
        """PL_ERR_ARG (raised) if a call since the last check met an index outside the map."""
        check(_track_lib().pl_map_check_indices(self._h))

    def set_keyframes(self, graph):
        """Upload the keyframe graph (pl_map_set_keyframes; keyframes numbered in ascending KeyFrame* address).  graph: dict(Tcw,
        Twc [K][4][4], bad [K] (optional), parent [K] (-1 none), and the CSR pairs pt_slot_offset / pt_slot, ln_slot_offset /
        ln_slot, cov_offset / cov, child_offset / child ([K + 1] offsets) and obs_offset [n_points + 1] / obs)."""
        Tcw = _f32(graph["Tcw"]).reshape(-1, 16)
        K = len(Tcw)
        a = dict(Tcw=Tcw, Twc=_f32(graph["Twc"]).reshape(-1, 16), parent=_i32(graph["parent"]))
        if graph.get("bad") is not None:
            a["bad"] = np.ascontiguousarray(graph["bad"], np.uint8)
        for k in ("pt_slot", "ln_slot", "cov", "child", "obs"):
            a[k + "_offset"] = _i32(graph[k + "_offset"]); a[k] = _i32(graph[k])
        self._graph = a
        d = PLKeyFrameGraphDesc(K, *[_p(a.get(f)) for f, _ in PLKeyFrameGraphDesc._fields_[1:]])
        check(_track_lib().pl_map_set_keyframes(self._h, C.byref(d)))

    def check_capacity(self):
        """PL_ERR_ARG (raised) if a local list outgrew its capacity since the last check."""
        check(_track_lib().pl_map_check_capacity(self._h))


def _local_struct(local, B, keep, to_dev):
    """local: dict(pt_index, pt_offset [B], pt_count [B], ln_index, ln_offset, ln_count, frames_since_reloc [B], max_frames,
    cap_local_points / cap_local_lines (default: the largest count))."""
    host = {k: np.ascontiguousarray(local[k], np.int32) for k in ("pt_offset", "pt_count", "ln_offset", "ln_count", "frames_since_reloc")}
    for k, v in host.items():
        assert v.shape == (B,), k
    keep.append(host)
    cLP = int(local.get("cap_local_points", max(int(host["pt_count"].max(initial=0)), 1)))
    cLL = int(local.get("cap_local_lines", max(int(host["ln_count"].max(initial=0)), 1)))
    arrs = [np.ascontiguousarray(local[k], np.int32).ravel() for k in ("pt_index", "ln_index")]
    idx = [to_dev(a) for a in arrs]
    keep.append(idx)
    s = PLTrackLocal(_p(host["pt_offset"]), _p(host["pt_count"]), idx[0][1], len(arrs[0]), cLP, _p(host["ln_offset"]), _p(host["ln_count"]),
                     idx[1][1], len(arrs[1]), cLL, _p(host["frames_since_reloc"]), int(local["max_frames"]))
    return s, cLP, cLL


def _out_shapes(B, cap, capL, cLP, cLL):
    return dict(Tcw=((B, 4, 4), np.float32), point_map=((B, cap), np.int32), point_outlier=((B, cap), np.uint8),
                line_map=((B, capL), np.int32), line_outlier=((B, capL), np.uint8), inliers=((B, 2), np.int32), ok=((B,), np.int32),
                pt_in_view=((B, cLP), np.uint8), pt_proj=((B, cLP, 2), np.float32), pt_level=((B, cLP), np.int32),
                pt_view_cos=((B, cLP), np.float32), ln_in_view=((B, cLL), np.uint8), ln_proj=((B, cLL, 4), np.float32),
                ln_level=((B, cLL), np.int32), ln_view_cos=((B, cLL), np.float32), pt_match=((B, cap), np.int32),
                ln_match=((B, capL), np.int32), prob_n_points=((B,), np.int32), prob_pt_obs=((B, cap, 2), np.float32),
                prob_pt_inv_sigma2=((B, cap), np.float32), prob_pt_Xw=((B, cap, 3), np.float32), prob_n_lines=((B,), np.int32),
                prob_line_func=((B, capL, 3), np.float64), prob_line_Xw=((B, capL, 6), np.float64))


def _torch_dev():
    import torch
    keep = []

    def to_dev(a):
        a = np.ascontiguousarray(a)
        t = torch.from_numpy(a.view(np.uint8).reshape(-1).copy() if a.size else np.zeros(16, np.uint8)).cuda()
        keep.append(t)
        return t, vp(t.data_ptr())
    return torch, keep, to_dev


def _run_dev(call, B, cap, capL, cLP, cLL, taps, keep, torch, scratch_query=None):
    shapes = _out_shapes(B, cap, capL, cLP, cLL)
    names = _TRACK_OUT if taps else _TRACK_OUT[:7]
    dev = {}
    for k in names:
        shp, dt = shapes[k]
        dev[k] = torch.zeros(max(int(np.prod(shp)) * np.dtype(dt).itemsize, 16), dtype=torch.uint8, device="cuda")
    o = PLTrackOut(*[vp(dev[k].data_ptr()) if k in dev else None for k in _TRACK_OUT])
    query = scratch_query or _track_lib().pl_track_local_map_scratch_bytes
    scratch = torch.empty(int(query(B, cap, capL, cLP, cLL)), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    check(call(o, vp(scratch.data_ptr())))
    torch.cuda.synchronize()
    out = {}
    for k in names:
        shp, dt = shapes[k]
        nb = int(np.prod(shp)) * np.dtype(dt).itemsize
        out[k] = dev[k][:nb].cpu().numpy().view(dt).reshape(shp)
    return out


def track_local_map(map, frames, local, taps=False, host=False, seen=None):
    """Tracking::TrackLocalMapWithLines (localisation mode) for B frames against `map` (pl_track_local_map_dev).

    frames: dict(keys_un [B][cap] KP_DTYPE, desc [B][cap][32], n [B], keylines [B][capL] KEYLINE_DTYPE, line_func [B][capL][3],
    line_desc [B][capL][32], nl [B], bounds [4], scale_factors, inv_level_sigma2, log_scale_factor, Tcw0 [B][4][4], K [B][4],
    point_map_in / line_map_in ([B][cap] map index or -1; optional)).  local: see _local_struct.
    Returns dict(Tcw, point_map, point_outlier, line_map, line_outlier, inliers [B][2], ok [B]) plus, with taps=True, the
    intermediates of PLTrackOut.  host=True (B = 1 only) calls the host-pointer entry pl_track_local_map instead.
    seen: dict with point_seen [B][cap] / line_seen [B][capL] (track_motion_model's outputs): the map entries the motion model
    discarded, skipped by the frustum test like held matches (pl_track_local_map_seen_dev); not with host=True."""
    L = _track_lib()
    B, cap = frames["keys_un"].shape[:2]
    capL = frames["keylines"].shape[1]
    nlev = len(frames["scale_factors"])
    arr = dict(keys_un=np.ascontiguousarray(frames["keys_un"], KP_DTYPE), desc=np.ascontiguousarray(frames["desc"], np.uint8),
               n=np.ascontiguousarray(frames["n"], np.int32), keylines=np.ascontiguousarray(frames["keylines"], KEYLINE_DTYPE),
               line_func=np.ascontiguousarray(frames["line_func"], np.float64), line_desc=np.ascontiguousarray(frames["line_desc"], np.uint8),
               nl=np.ascontiguousarray(frames["nl"], np.int32), bounds=_f32(frames["bounds"]), scale_factors=_f32(frames["scale_factors"]),
               inv_level_sigma2=_f32(frames["inv_level_sigma2"]), Tcw0=_f32(frames["Tcw0"]).reshape(B, 16), K=_f32(frames["K"]).reshape(B, 4))
    for k in ("point_map_in", "line_map_in"):
        if frames.get(k) is not None:
            arr[k] = np.ascontiguousarray(frames[k], np.int32)
    if host:
        assert B == 1
        if seen is not None:
            raise ValueError("track_local_map: seen= needs the device entry (host=False)")
        keep = []
        s, cLP, cLL = _local_struct(local, 1, keep, lambda a: (a, _p(a)))
        F = PLTrackFrames(1, _p(arr["keys_un"]), _p(arr["desc"]), _p(arr["n"]), cap, _p(arr["keylines"]), _p(arr["line_func"]),
                          _p(arr["line_desc"]), _p(arr["nl"]), capL, _p(arr["bounds"]), _p(arr["scale_factors"]), _p(arr["inv_level_sigma2"]),
                          nlev, float(frames["log_scale_factor"]), _p(arr["Tcw0"]), _p(arr["K"]), _p(arr.get("point_map_in")),
                          _p(arr.get("line_map_in")))
        n, nl = int(arr["n"][0]), int(arr["nl"][0])
        lp, ll = int(s.cap_local_points), int(s.cap_local_lines)
        shapes = _out_shapes(1, cap, capL, lp, ll)
        out = {k: np.zeros(shp, dt) for k, (shp, dt) in shapes.items()}
        names = _TRACK_OUT if taps else _TRACK_OUT[:7]
        o = PLTrackOut(*[_p(out[k]) if (k in names and k != "ok") else None for k in _TRACK_OUT])
        out["ok"][0] = check(L.pl_track_local_map(map._h, C.byref(F), C.byref(s), C.byref(o)))
        return {k: out[k] for k in names}
    torch, keep, to_dev = _torch_dev()
    d = {k: to_dev(v)[1] for k, v in arr.items()}
    s, cLP, cLL = _local_struct(local, B, keep, to_dev)
    F = PLTrackFrames(B, d["keys_un"], d["desc"], d["n"], cap, d["keylines"], d["line_func"], d["line_desc"], d["nl"], capL, d["bounds"],
                      d["scale_factors"], d["inv_level_sigma2"], nlev, float(frames["log_scale_factor"]), d["Tcw0"], d["K"],
                      d.get("point_map_in"), d.get("line_map_in"))
    if seen is None:
        call = lambda o, scr: L.pl_track_local_map_dev(map._h, C.byref(F), C.byref(s), C.byref(o), scr, None)   # noqa: E731
    else:
        ps = to_dev(np.ascontiguousarray(seen["point_seen"], np.int32).reshape(B, cap))[1]
        ls = to_dev(np.ascontiguousarray(seen["line_seen"], np.int32).reshape(B, capL))[1]
        call = lambda o, scr: L.pl_track_local_map_seen_dev(map._h, C.byref(F), ps, ls, C.byref(s), C.byref(o), scr, None)   # noqa: E731
    out = _run_dev(call, B, cap, capL, cLP, cLL, taps, keep, torch)
    map.check_indices()
    return out


def _frontend_track_local_map(self, map, Tcw0, K, local, point_map_in=None, line_map_in=None, taps=False):
    """Tracking::TrackLocalMapWithLines on the features of the last run() / run_dev() (pl_frontend_track_local_map_dev): frames
    0..B-1 of that step, B = len(Tcw0).  point_map_in / line_map_in are [B][capK] / [B][capL] (map index or -1) or None."""
    L = _track_lib()
    B = len(Tcw0)
    torch, keep, to_dev = _torch_dev()
    T0 = to_dev(_f32(Tcw0).reshape(B, 16))[1]; Kd = to_dev(_f32(K).reshape(B, 4))[1]
    pm = None if point_map_in is None else to_dev(np.ascontiguousarray(point_map_in, np.int32).reshape(B, self.capK))[1]
    lm = None if line_map_in is None else to_dev(np.ascontiguousarray(line_map_in, np.int32).reshape(B, self.capL))[1]
    s, cLP, cLL = _local_struct(local, B, keep, to_dev)
    out = _run_dev(lambda o, scr: L.pl_frontend_track_local_map_dev(self._h, map._h, B, T0, Kd, pm, lm, C.byref(s), C.byref(o), scr, None),
                   B, self.capK, self.capL, cLP, cLL, taps, keep, torch)
    map.check_indices()
    return out


Frontend.track_local_map = _frontend_track_local_map


# ---------------------------------------------------------------------------------------------- the constant-velocity motion model
class PLTrackLast(C.Structure):
    _fields_ = [(k, vp) for k in ("keys_un", "n", "keylines", "nl", "point_map", "point_outlier", "line_map", "line_outlier", "Tcw",
                                  "velocity")]


_MM_OUT = ["Tcw", "point_map", "line_map", "point_seen", "line_seen", "nmatches", "ok", "vo", "guess", "pt_match", "pt_match_retry",
           "retried", "ln_match", "ln_in_view", "ln_proj", "ln_level", "ln_view_cos", "prob_n_points", "prob_pt_obs", "prob_pt_inv_sigma2",
           "prob_pt_Xw", "prob_n_lines", "prob_line_func", "prob_line_Xw"]


class PLTrackMotionOut(C.Structure):
    _fields_ = [(k, vp) for k in _MM_OUT]


def _mm_shapes(B, cap, capL):
    return dict(Tcw=((B, 4, 4), np.float32), point_map=((B, cap), np.int32), line_map=((B, capL), np.int32), point_seen=((B, cap), np.int32),
                line_seen=((B, capL), np.int32), nmatches=((B, 2), np.int32), ok=((B,), np.int32), vo=((B,), np.int32),
                guess=((B, 4, 4), np.float32), pt_match=((B, cap), np.int32), pt_match_retry=((B, cap), np.int32), retried=((B,), np.uint8),
                ln_match=((B, capL), np.int32), ln_in_view=((B, capL), np.uint8), ln_proj=((B, capL, 4), np.float32),
                ln_level=((B, capL), np.int32), ln_view_cos=((B, capL), np.float32), prob_n_points=((B,), np.int32),
                prob_pt_obs=((B, cap, 2), np.float32), prob_pt_inv_sigma2=((B, cap), np.float32), prob_pt_Xw=((B, cap, 3), np.float32),
                prob_n_lines=((B,), np.int32), prob_line_func=((B, capL, 3), np.float64), prob_line_Xw=((B, capL, 6), np.float64))


def track_motion_model(map, frames, last, taps=False, host=False):
    """Tracking::TrackWithMotionModel (monocular, localisation mode) for B frames against `map` (pl_track_motion_model_dev).

    frames: as for track_local_map, without Tcw0 / point_map_in / line_map_in.  last: dict(keys_un [B][cap], n [B], keylines
    [B][capL], nl [B], point_map / point_outlier [B][cap], line_map / line_outlier [B][capL], Tcw [B][4][4] (after UpdateLastFrame),
    velocity [B][4][4], vo [B] (optional, the mbVO passed in; default 0)), with the caps of `frames`.
    Returns dict(Tcw, point_map, line_map, point_seen, line_seen, nmatches [B][2], ok [B], vo [B]) plus, with taps=True, the
    intermediates of PLTrackMotionOut.  host=True (B = 1 only) calls the host-pointer entry pl_track_motion_model instead."""
    L = _track_lib()
    B, cap = frames["keys_un"].shape[:2]
    capL = frames["keylines"].shape[1]
    assert last["keys_un"].shape[:2] == (B, cap) and last["keylines"].shape[:2] == (B, capL)
    nlev = len(frames["scale_factors"])
    arr = dict(keys_un=np.ascontiguousarray(frames["keys_un"], KP_DTYPE), desc=np.ascontiguousarray(frames["desc"], np.uint8),
               n=np.ascontiguousarray(frames["n"], np.int32), keylines=np.ascontiguousarray(frames["keylines"], KEYLINE_DTYPE),
               line_func=np.ascontiguousarray(frames["line_func"], np.float64), line_desc=np.ascontiguousarray(frames["line_desc"], np.uint8),
               nl=np.ascontiguousarray(frames["nl"], np.int32), bounds=_f32(frames["bounds"]), scale_factors=_f32(frames["scale_factors"]),
               inv_level_sigma2=_f32(frames["inv_level_sigma2"]), K=_f32(frames["K"]).reshape(B, 4),
               l_keys_un=np.ascontiguousarray(last["keys_un"], KP_DTYPE), l_n=np.ascontiguousarray(last["n"], np.int32),
               l_keylines=np.ascontiguousarray(last["keylines"], KEYLINE_DTYPE), l_nl=np.ascontiguousarray(last["nl"], np.int32),
               l_point_map=np.ascontiguousarray(last["point_map"], np.int32), l_point_outlier=np.ascontiguousarray(last["point_outlier"], np.uint8),
               l_line_map=np.ascontiguousarray(last["line_map"], np.int32), l_line_outlier=np.ascontiguousarray(last["line_outlier"], np.uint8),
               l_Tcw=_f32(last["Tcw"]).reshape(B, 16), l_velocity=_f32(last["velocity"]).reshape(B, 16))
    vo_in = np.ascontiguousarray(last.get("vo", np.zeros(B)), np.int32).reshape(B)
    shapes = _mm_shapes(B, cap, capL)
    names = _MM_OUT if taps else _MM_OUT[:8]

    def structs(d):
        F = PLTrackFrames(B, d["keys_un"], d["desc"], d["n"], cap, d["keylines"], d["line_func"], d["line_desc"], d["nl"], capL, d["bounds"],
                          d["scale_factors"], d["inv_level_sigma2"], nlev, float(frames["log_scale_factor"]), None, d["K"], None, None)
        Ls = PLTrackLast(*[d["l_" + k] for k, _ in PLTrackLast._fields_])
        return F, Ls
    if host:
        assert B == 1
        F, Ls = structs({k: _p(v) for k, v in arr.items()})
        out = {k: np.zeros(shp, dt) for k, (shp, dt) in shapes.items()}
        out["vo"][:] = vo_in
        o = PLTrackMotionOut(*[_p(out[k]) if (k in names and k != "ok") else None for k in _MM_OUT])
        out["ok"][0] = check(L.pl_track_motion_model(map._h, C.byref(F), C.byref(Ls), C.byref(o)))
        return {k: out[k] for k in names}
    torch, keep, to_dev = _torch_dev()
    F, Ls = structs({k: to_dev(v)[1] for k, v in arr.items()})
    dev = {}
    for k in names:
        shp, dt = shapes[k]
        dev[k] = torch.zeros(max(int(np.prod(shp)) * np.dtype(dt).itemsize, 16), dtype=torch.uint8, device="cuda")
    dev["vo"][:4 * B].copy_(torch.from_numpy(vo_in.view(np.uint8)))
    o = PLTrackMotionOut(*[vp(dev[k].data_ptr()) if k in dev else None for k in _MM_OUT])
    scratch = torch.empty(int(L.pl_track_motion_model_scratch_bytes(B, cap, capL)), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    check(L.pl_track_motion_model_dev(map._h, C.byref(F), C.byref(Ls), C.byref(o), vp(scratch.data_ptr()), None))
    torch.cuda.synchronize()
    out = {}
    for k in names:
        shp, dt = shapes[k]
        out[k] = dev[k][:int(np.prod(shp)) * np.dtype(dt).itemsize].cpu().numpy().view(dt).reshape(shp)
    map.check_indices()
    return out


def track_velocity(Tcw, Tcw_last, ok, velocity):
    """mVelocity = mCurrentFrame.mTcw * LastTwc for B frames (pl_track_velocity_dev): returns `velocity` [B][4][4] with the frames
    where ok[b] replaced."""
    import torch
    B = len(Tcw)
    L = _track_lib()
    t = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in
         (_f32(Tcw).reshape(B, 16), _f32(Tcw_last).reshape(B, 16), np.ascontiguousarray(ok, np.int32).reshape(B),
          _f32(velocity).reshape(B, 16).copy())]
    torch.cuda.synchronize()
    check(L.pl_track_velocity_dev(B, *[vp(x.data_ptr()) for x in t], None))
    torch.cuda.synchronize()
    return t[3].cpu().numpy().reshape(B, 4, 4)


# ---------------------------------------------------------------------------------------------- the local map from the keyframe graph
class PLKeyFrameGraphDesc(C.Structure):
    _fields_ = [("n_kf", C.c_int)] + [(k, vp) for k in ("Tcw", "Twc", "bad", "parent", "pt_slot_offset", "pt_slot", "ln_slot_offset",
                                                        "ln_slot", "cov_offset", "cov", "child_offset", "child", "obs_offset", "obs")]


class PLLocalMap(C.Structure):
    _fields_ = [("kf", vp), ("n_kf", vp), ("cap_kf", C.c_int), ("ref_kf", vp), ("pt_index", vp), ("pt_count", vp),
                ("cap_local_points", C.c_int), ("ln_index", vp), ("ln_count", vp), ("cap_local_lines", C.c_int)]


def _local_map_struct(t, cap_kf, cLP, cLL):
    """t: dict of torch tensors kf, n_kf, ref_kf, pt_index, pt_count, ln_index, ln_count."""
    a = {k: vp(v.data_ptr()) for k, v in t.items()}
    return PLLocalMap(a["kf"], a["n_kf"], cap_kf, a["ref_kf"], a["pt_index"], a["pt_count"], cLP, a["ln_index"], a["ln_count"], cLL)


def _opt_dev(a, B, to_dev):
    return None if a is None else to_dev(np.ascontiguousarray(a, np.int32).reshape(B))[1]


def update_local_map(map, point_map, kf, n_kf, ref_kf, cap_local_points, cap_local_lines, ok=None, vo=None):
    """Tracking::UpdateLocalMap for B frames (pl_track_update_local_map_dev) on point_map [B][cap] (map index or -1).
    kf [B][cap_kf], n_kf [B] and ref_kf [B] are the local keyframe lists and reference keyframes passed in (kept by a frame whose
    matches vote for no keyframe); ok / vo (optional [B]): frame b runs only if ok[b] and not vo[b].  Returns dict(kf, n_kf, ref_kf,
    pt_index [B][cap_local_points], pt_count [B], ln_index [B][cap_local_lines], ln_count [B]); counts are the true sizes, entries
    past a capacity are left 0 and Map.check_capacity() raises."""
    import torch
    point_map = np.ascontiguousarray(point_map, np.int32)
    B, cap = point_map.shape
    kf = np.ascontiguousarray(kf, np.int32).reshape(B, -1)
    _, keep, to_dev = _torch_dev()
    t = dict(kf=torch.from_numpy(kf.copy()).cuda(), n_kf=torch.from_numpy(_i32(n_kf).reshape(B).copy()).cuda(),
             ref_kf=torch.from_numpy(_i32(ref_kf).reshape(B).copy()).cuda(),
             pt_index=torch.zeros((B, cap_local_points), dtype=torch.int32, device="cuda"), pt_count=torch.zeros(B, dtype=torch.int32, device="cuda"),
             ln_index=torch.zeros((B, cap_local_lines), dtype=torch.int32, device="cuda"), ln_count=torch.zeros(B, dtype=torch.int32, device="cuda"))
    s = _local_map_struct(t, kf.shape[1], cap_local_points, cap_local_lines)
    pm = to_dev(point_map)[1]
    torch.cuda.synchronize()
    check(_track_lib().pl_track_update_local_map_dev(map._h, B, pm, cap, _opt_dev(ok, B, to_dev), _opt_dev(vo, B, to_dev), C.byref(s), None))
    torch.cuda.synchronize()
    out = {k: v.cpu().numpy() for k, v in t.items()}
    map.check_indices()
    return out


def track_local_map_lists(map, frames, local, frames_since_reloc, max_frames, taps=False, seen=None, ok=None, vo=None):
    """track_local_map on device lists (pl_track_local_map_lists_dev): local = dict(pt_index [B][cap_local_points], pt_count [B],
    ln_index [B][cap_local_lines], ln_count [B]) as update_local_map returns them (counts over a capacity are clamped);
    frames_since_reloc [B]; ok / vo (optional [B]) gate the frames: a frame gated off passes through (Tcw = Tcw0, held matches
    kept, outlier flags 0, ok = ok[b])."""
    L = _track_lib()
    B, cap = frames["keys_un"].shape[:2]
    capL = frames["keylines"].shape[1]
    nlev = len(frames["scale_factors"])
    arr = dict(keys_un=np.ascontiguousarray(frames["keys_un"], KP_DTYPE), desc=np.ascontiguousarray(frames["desc"], np.uint8),
               n=np.ascontiguousarray(frames["n"], np.int32), keylines=np.ascontiguousarray(frames["keylines"], KEYLINE_DTYPE),
               line_func=np.ascontiguousarray(frames["line_func"], np.float64), line_desc=np.ascontiguousarray(frames["line_desc"], np.uint8),
               nl=np.ascontiguousarray(frames["nl"], np.int32), bounds=_f32(frames["bounds"]), scale_factors=_f32(frames["scale_factors"]),
               inv_level_sigma2=_f32(frames["inv_level_sigma2"]), Tcw0=_f32(frames["Tcw0"]).reshape(B, 16), K=_f32(frames["K"]).reshape(B, 4))
    for k in ("point_map_in", "line_map_in"):
        if frames.get(k) is not None:
            arr[k] = np.ascontiguousarray(frames[k], np.int32)
    torch, keep, to_dev = _torch_dev()
    d = {k: to_dev(v)[1] for k, v in arr.items()}
    F = PLTrackFrames(B, d["keys_un"], d["desc"], d["n"], cap, d["keylines"], d["line_func"], d["line_desc"], d["nl"], capL, d["bounds"],
                      d["scale_factors"], d["inv_level_sigma2"], nlev, float(frames["log_scale_factor"]), d["Tcw0"], d["K"],
                      d.get("point_map_in"), d.get("line_map_in"))
    pi = np.ascontiguousarray(local["pt_index"], np.int32).reshape(B, -1); li = np.ascontiguousarray(local["ln_index"], np.int32).reshape(B, -1)
    cLP, cLL = pi.shape[1], li.shape[1]
    one = to_dev(np.zeros(B, np.int32))[1]
    s = PLLocalMap(one, one, 1, one, to_dev(pi)[1], _opt_dev(local["pt_count"], B, to_dev), cLP, to_dev(li)[1],
                   _opt_dev(local["ln_count"], B, to_dev), cLL)
    since = _opt_dev(frames_since_reloc, B, to_dev)
    ps = ls = None
    if seen is not None:
        ps = to_dev(np.ascontiguousarray(seen["point_seen"], np.int32).reshape(B, cap))[1]
        ls = to_dev(np.ascontiguousarray(seen["line_seen"], np.int32).reshape(B, capL))[1]
    okd, vod = _opt_dev(ok, B, to_dev), _opt_dev(vo, B, to_dev)
    out = _run_dev(lambda o, scr: L.pl_track_local_map_lists_dev(map._h, C.byref(F), ps, ls, C.byref(s), since, int(max_frames), okd, vod,
                                                                 C.byref(o), scr, None),
                   B, cap, capL, cLP, cLL, taps, keep, torch, L.pl_track_local_map_lists_scratch_bytes)
    map.check_indices()
    return out


def _ref_pose(fn, map, P, ref_kf, out=None):
    import torch
    B = len(ref_kf)
    t = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in
         (_f32(P).reshape(B, 16), _i32(ref_kf).reshape(B), np.zeros((B, 16), np.float32) if out is None else _f32(out).reshape(B, 16).copy())]
    torch.cuda.synchronize()
    check(fn(map._h, B, *[vp(x.data_ptr()) for x in t], None))
    torch.cuda.synchronize()
    return t[2].cpu().numpy().reshape(B, 4, 4)


def relative_pose(map, Tcw, ref_kf, out=None):
    """Tcr = Tcw * Twc[ref_kf] for B frames (pl_track_relative_pose_dev, Tracking.cc:582).  A frame whose ref_kf is outside the
    graph keeps `out`'s value (zeros if None) and Map.check_indices() raises."""
    return _ref_pose(_track_lib().pl_track_relative_pose_dev, map, Tcw, ref_kf, out)


def last_pose(map, Tcr, ref_kf, out=None):
    """mLastFrame.mTcw = Tcr * Tcw[ref_kf] for B frames (pl_track_last_pose_dev, the monocular UpdateLastFrame, :1242-1245)."""
    return _ref_pose(_track_lib().pl_track_last_pose_dev, map, Tcr, ref_kf, out)


class LocalizationChain:
    """The OK-state localisation frame for B independent streams against a fixed map with its keyframe graph, every buffer on the
    device and allocated once, so that localization_step() only enqueues work (it may be captured into a CUDA graph):

        last pose -> motion model -> update local map -> local-map step -> velocity -> relative pose

    set_frames() uploads the current frames' features; set_state() the streams' state (the last frames, as TrackLocalMapWithLines
    left them, Tcr, ref_kf, velocity, vo, the local keyframe lists).  After a step, fetch() returns every stage's outputs; the
    current frames have become the last frames.  frames_since_reloc [B] (device tensor) is the caller's to update."""

    def __init__(self, map, B, cap, capL, cap_kf, cap_local_points, cap_local_lines, bounds, scale_factors, inv_level_sigma2,
                 log_scale_factor, max_frames=30):
        import torch
        self.map, self.B, self.cap, self.capL, self.cap_kf, self.cLP, self.cLL = map, B, cap, capL, cap_kf, cap_local_points, cap_local_lines
        self.max_frames, self.log_scale_factor, self.nlev = int(max_frames), float(log_scale_factor), len(scale_factors)
        dev = dict(device="cuda")
        z = lambda shape, dt: torch.zeros(shape, dtype=dt, **dev)   # noqa: E731
        u8, i32, f32, f64 = torch.uint8, torch.int32, torch.float32, torch.float64
        kp, kl = np.dtype(KP_DTYPE).itemsize, np.dtype(KEYLINE_DTYPE).itemsize
        self.tab = {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in
                    (("bounds", _f32(bounds)), ("scale_factors", _f32(scale_factors)), ("inv_level_sigma2", _f32(inv_level_sigma2)))}
        self.cur = dict(keys_un=z((B, cap * kp), u8), desc=z((B, cap, 32), u8), n=z(B, i32), keylines=z((B, capL * kl), u8),
                        line_func=z((B, capL, 3), f64), line_desc=z((B, capL, 32), u8), nl=z(B, i32), K=z((B, 4), f32))
        self.last = dict(keys_un=z((B, cap * kp), u8), n=z(B, i32), keylines=z((B, capL * kl), u8), nl=z(B, i32), point_map=z((B, cap), i32),
                         point_outlier=z((B, cap), u8), line_map=z((B, capL), i32), line_outlier=z((B, capL), u8), Tcw=z((B, 16), f32),
                         velocity=z((B, 16), f32))
        self.state = dict(Tcr=z((B, 16), f32), vo=z(B, i32), frames_since_reloc=z(B, i32))
        self.local = dict(kf=z((B, cap_kf), i32), n_kf=z(B, i32), ref_kf=z(B, i32), pt_index=z((B, cap_local_points), i32),
                          pt_count=z(B, i32), ln_index=z((B, cap_local_lines), i32), ln_count=z(B, i32))
        self.mm = {k: z(((B,) + shp[1:]) if len(shp) > 1 else B, getattr(torch, np.dtype(dt).name)) for k, (shp, dt) in
                   _mm_shapes(B, cap, capL).items() if k in _MM_OUT[:8]}
        self.mm["vo"] = self.state["vo"]                                       # mbVO is in / out
        sh = _out_shapes(B, cap, capL, cap_local_points, cap_local_lines)
        self.lo = {k: z(sh[k][0], getattr(torch, np.dtype(sh[k][1]).name)) for k in _TRACK_OUT[:7]}
        L = _track_lib()
        self.mm_scratch = torch.empty(int(L.pl_track_motion_model_scratch_bytes(B, cap, capL)), dtype=u8, **dev)
        self.lo_scratch = torch.empty(int(L.pl_track_local_map_lists_scratch_bytes(B, cap, capL, cap_local_points, cap_local_lines)),
                                      dtype=u8, **dev)
        p = lambda t: vp(t.data_ptr())   # noqa: E731
        c, la, tb = self.cur, self.last, self.tab

        def frames(Tcw0, pm, lm):
            return PLTrackFrames(B, p(c["keys_un"]), p(c["desc"]), p(c["n"]), cap, p(c["keylines"]), p(c["line_func"]), p(c["line_desc"]),
                                 p(c["nl"]), capL, p(tb["bounds"]), p(tb["scale_factors"]), p(tb["inv_level_sigma2"]), self.nlev,
                                 self.log_scale_factor, Tcw0, p(c["K"]), pm, lm)
        self._F_mm = frames(None, None, None)
        self._F_lo = frames(p(self.mm["Tcw"]), p(self.mm["point_map"]), p(self.mm["line_map"]))
        self._last = PLTrackLast(*[p(la[k]) for k, _ in PLTrackLast._fields_])
        self._mm_out = PLTrackMotionOut(*[p(self.mm[k]) if k in self.mm else None for k in _MM_OUT])
        self._lo_out = PLTrackOut(*[p(self.lo[k]) if k in self.lo else None for k in _TRACK_OUT])
        self._local = _local_map_struct(self.local, cap_kf, cap_local_points, cap_local_lines)

    def set_frames(self, frames):
        """frames: the current frames as for track_motion_model (keys_un, desc, n, keylines, line_func, line_desc, nl, K)."""
        import torch
        for k in ("keys_un", "desc", "n", "keylines", "line_func", "line_desc", "nl", "K"):
            a = np.ascontiguousarray(frames[k])
            self.cur[k].copy_(torch.from_numpy(a.view(np.uint8).reshape(self.cur[k].shape) if a.dtype.fields else
                                               a.astype(np.dtype(str(self.cur[k].dtype).replace("torch.", ""))).reshape(self.cur[k].shape)))

    def set_state(self, last, Tcr, ref_kf, velocity, kf, n_kf, vo=None, frames_since_reloc=None):
        """last: the last frames as for track_motion_model (keys_un, n, keylines, nl, point_map, point_outlier, line_map,
        line_outlier); Tcr [B][4][4] and ref_kf [B] of the last frames; velocity [B][4][4]; kf [B][cap_kf] / n_kf [B] the local
        keyframe lists."""
        import torch
        B = self.B
        put = lambda t, a: t.copy_(torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(t.shape) if np.asarray(a).dtype.fields   # noqa: E731
                                                   else np.ascontiguousarray(a).astype(np.dtype(str(t.dtype).replace("torch.", ""))).reshape(t.shape)))
        for k in ("keys_un", "n", "keylines", "nl", "point_map", "point_outlier", "line_map", "line_outlier"):
            put(self.last[k], last[k])
        put(self.last["velocity"], _f32(velocity).reshape(B, 16)); put(self.state["Tcr"], _f32(Tcr).reshape(B, 16))
        put(self.local["ref_kf"], _i32(ref_kf)); put(self.local["kf"], _i32(kf)); put(self.local["n_kf"], _i32(n_kf))
        put(self.state["vo"], np.zeros(B, np.int32) if vo is None else _i32(vo))
        put(self.state["frames_since_reloc"], np.full(B, 1 << 20, np.int32) if frames_since_reloc is None else _i32(frames_since_reloc))

    def localization_step(self, stream=None):
        """Enqueue one frame of every stream on `stream` (a torch.cuda.Stream; default the current stream).  No host
        synchronisation and no host-to-device copy: only kernels and device-to-device copies."""
        import torch
        st = stream or torch.cuda.current_stream()
        h = vp(st.cuda_stream or 1)      # the default stream as cudaStreamLegacy: NULL would select the map's own stream

        L, M, B, p = _track_lib(), self.map._h, self.B, (lambda t: vp(t.data_ptr()))
        la, mm, lo, loc = self.last, self.mm, self.lo, self.local
        check(L.pl_track_last_pose_dev(M, B, p(self.state["Tcr"]), p(loc["ref_kf"]), p(la["Tcw"]), h))
        check(L.pl_track_motion_model_dev(M, C.byref(self._F_mm), C.byref(self._last), C.byref(self._mm_out), p(self.mm_scratch), h))
        check(L.pl_track_update_local_map_dev(M, B, p(mm["point_map"]), self.cap, p(mm["ok"]), p(mm["vo"]), C.byref(self._local), h))
        check(L.pl_track_local_map_lists_dev(M, C.byref(self._F_lo), p(mm["point_seen"]), p(mm["line_seen"]), C.byref(self._local),
                                             p(self.state["frames_since_reloc"]), self.max_frames, p(mm["ok"]), p(mm["vo"]),
                                             C.byref(self._lo_out), p(self.lo_scratch), h))
        check(L.pl_track_velocity_dev(B, p(lo["Tcw"]), p(la["Tcw"]), p(lo["ok"]), p(la["velocity"]), h))
        check(L.pl_track_relative_pose_dev(M, B, p(lo["Tcw"]), p(loc["ref_kf"]), p(self.state["Tcr"]), h))
        # the current frames become the last frames (mLastFrame = Frame(mCurrentFrame))
        with torch.cuda.stream(st):
            for k in ("keys_un", "n", "keylines", "nl"):
                la[k].copy_(self.cur[k])
            for k in ("point_map", "point_outlier", "line_map", "line_outlier"):
                la[k].copy_(lo[k])

    def fetch(self):
        """Every stage's outputs as numpy: Tlast (the last pose of this step), mm (motion model), local (the local map), lo (the
        local-map step), velocity and Tcr."""
        import torch
        torch.cuda.synchronize()
        B = self.B
        n = lambda t: t.cpu().numpy()   # noqa: E731
        mm = {k: n(v) for k, v in self.mm.items()}
        mm["Tcw"] = mm["Tcw"].reshape(B, 4, 4)
        lo = {k: n(v) for k, v in self.lo.items()}
        lo["Tcw"] = lo["Tcw"].reshape(B, 4, 4)
        return dict(Tlast=n(self.last["Tcw"]).reshape(B, 4, 4), mm=mm, local={k: n(v) for k, v in self.local.items()}, lo=lo,
                    velocity=n(self.last["velocity"]).reshape(B, 4, 4), Tcr=n(self.state["Tcr"]).reshape(B, 4, 4))
