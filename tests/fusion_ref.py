"""Float CPU oracle of the RGB-D fusion chain (tests/native/fusion_oracle.cpp, built by __graft_entry__.build()) and the inputs the
fusion tests share: a scene's rendered depth frames, colour frames and float poses in both directions."""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        path = os.path.join(_HERE, "native", "libfusion_oracle.so")
        if not os.path.exists(path):
            raise RuntimeError(f"{path} not found: run __graft_entry__.build()")
        L = C.CDLL(path)
        L.fo_create.restype = C.c_void_p
        L.fo_create.argtypes = [C.c_void_p, C.c_int, C.c_int]
        L.fo_clone.restype = C.c_void_p
        L.fo_clone.argtypes = [C.c_void_p]
        L.fo_destroy.argtypes = [C.c_void_p]
        L.fo_integrate.argtypes = [C.c_void_p, C.c_int] + [C.c_void_p] * 8
        L.fo_finish.argtypes = [C.c_void_p, C.c_int]
        L.fo_num.restype = C.c_int64
        L.fo_num.argtypes = [C.c_void_p]
        L.fo_volume.argtypes = [C.c_void_p] + [C.c_void_p] * 4
        L.fo_erode.argtypes = [C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
        L.fo_normals.argtypes = [C.c_void_p] * 4
        L.fo_bounds.argtypes = [C.c_void_p, C.c_void_p, C.c_float, C.c_float, C.c_float, C.c_void_p, C.c_void_p]
        _LIB = L
    return _LIB


def _a(x, t):
    return np.ascontiguousarray(x, t)


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def cam_arrays(cam):
    """cam: (W, H, fx, fy, cx, cy) -> (int32[2], float32[4])."""
    return _a(cam[:2], np.int32), _a(cam[2:], np.float32)


class FusionOracle:
    def __init__(self, voxel_size=0.004, depth_min=0.1, depth_max=4.0, weight_sample=10.0, clip=(0.0,) * 6, window=2, iterations=10):
        self.pf = _a([voxel_size, depth_min, depth_max, weight_sample, *clip], np.float32)
        self.h = lib().fo_create(_ptr(self.pf), int(window), int(iterations))

    def __del__(self):
        if getattr(self, "h", None):
            lib().fo_destroy(self.h)
            self.h = None

    def clone(self):
        o = FusionOracle.__new__(FusionOracle)
        o.pf = self.pf
        o.h = lib().fo_clone(self.h)
        return o

    def integrate(self, depth_cam, depth, color_cam, bgr, c2w, w2c):
        dwh, dk = cam_arrays(depth_cam)
        cwh, ck = cam_arrays(color_cam)
        depth, bgr = _a(depth, np.float32), _a(bgr, np.uint8)
        c2w, w2c = _a(c2w, np.float32), _a(w2c, np.float32)
        return lib().fo_integrate(self.h, int(depth.shape[0]), _ptr(dwh), _ptr(dk), _ptr(depth), _ptr(cwh), _ptr(ck), _ptr(bgr), _ptr(c2w), _ptr(w2c))

    def finish(self, mode: int) -> int:
        """mode 1: correctSDF as Jacobi sweeps, 2: Gauss-Seidel in canonical order, 0: none; then clearInvalidVoxels.  Returns sweeps."""
        return int(lib().fo_finish(self.h, int(mode)))

    def volume(self):
        n = int(lib().fo_num(self.h))
        out = dict(xyz=np.empty((n, 3), np.int32), sdf=np.empty(n, np.float32), weight=np.empty(n, np.float32), rgb=np.empty((n, 3), np.uint8))
        if n:
            lib().fo_volume(self.h, _ptr(out["xyz"]), _ptr(out["sdf"]), _ptr(out["weight"]), _ptr(out["rgb"]))
        return out


def erode(depth, window):
    d = _a(depth, np.float32)
    out = np.empty_like(d)
    lib().fo_erode(d.shape[1], d.shape[0], int(window), _ptr(d), _ptr(out))
    return out


def normals(cam, depth):
    wh, k = cam_arrays(cam)
    d = _a(depth, np.float32)
    out = np.empty(d.shape + (3,), np.float32)
    lib().fo_normals(_ptr(wh), _ptr(k), _ptr(d), _ptr(out))
    return out


def bounds(cam, dmin, dmax, vs, rt):
    wh, k = cam_arrays(cam)
    rt = _a(rt, np.float32)
    b = np.empty(6, np.int32)
    lib().fo_bounds(_ptr(wh), _ptr(k), dmin, dmax, vs, _ptr(rt), _ptr(b))
    return b


def scene_inputs(s):
    """Depth camera, depth [F,H,W], colour camera (= depth camera), BGR frames and float poses camera->world / world->camera of a
    synthetic scene (its true poses)."""
    from intrinsic3d_b200.scene import aa_to_rotation, make_color_frames
    F, H, W = s["depth"].shape
    fx, fy, cx, cy = (float(v) for v in s["intr"])
    cam = (W, H, fx, fy, cx, cy)
    c2w = np.empty((F, 12), np.float32)
    w2c = np.empty((F, 12), np.float32)
    for f in range(F):
        R = aa_to_rotation(s["poses_true"][f, :3])
        t = s["poses_true"][f, 3:]
        w2c[f, :9] = R.reshape(-1); w2c[f, 9:] = t
        c2w[f, :9] = R.T.reshape(-1); c2w[f, 9:] = -R.T @ t
    return cam, np.ascontiguousarray(s["depth"], np.float32), cam, make_color_frames(s), c2w, w2c


def depth_range(s):
    """A depth range that holds the whole rendered object."""
    d = s["depth"][s["depth"] > 0]
    return float(np.floor(d.min() * 10) / 10), float(np.ceil(d.max() * 10) / 10 + 0.1)
