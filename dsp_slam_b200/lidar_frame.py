"""A KITTI LiDAR keyframe's object detections built on the H100 (libdspgn's DspgnLidarFrame).

    LidarFrameBuilder(K, T_cam_velo, configs, img_hw).detections(velo_pts, detections_3d, masks_2d, bboxes_2d)
    KITIISequence(data_dir, configs).get_frame_by_id(frame_id)        reconstruct/kitti_sequence.py:219-260

`detections` returns the instance list of the reference's FrameWithLiDAR.get_detections
(reconstruct/kitti_sequence.py:99-216), bit for bit, as ResultDicts in depth order with the attributes the Tracking
thread (src/Tracking_util.cc:37-50) and reconstruct_frame.py read: T_cam_obj, surface_points, rays (None or array),
depth, scale, num_surface_points, is_front, and, for a matched box, mask and bbox (views of the caller's arrays).
The per-box 4x4 matrices and the depth order stay on the host (numpy's float32 cos and LAPACK's inverse); the scan
geometry, the mask association, the background sampler and the rays run on the device in one call.  The occlusion
mask of the reference is not built: nothing reads it.
"""
import ctypes as C
import os
import sys

import numpy as np

from . import _lib
from .optimizer import ResultDict, _cfg_get, _warn_once


def _np(a):
    """numpy view of an array or a CPU torch tensor (torch.load of the stored labels gives either)."""
    if isinstance(a, np.ndarray):
        return a
    if hasattr(a, "detach"):
        return a.detach().cpu().numpy()
    return np.asarray(a)


def _box_matrices(det):
    """T_velo_obj and T_obj_velo of one box row (x, y, z, w, l, h, theta), as kitti_sequence.py:118-122 builds them."""
    trans, size, theta = det[:3], det[3:6], det[6]
    c, s = np.cos(theta), np.sin(theta)
    T_velo_obj = np.array([[c, 0, -s, trans[0]],
                           [-s, 0, -c, trans[1]],
                           [0, 1, 0, trans[2] + size[2] / 2],
                           [0, 0, 0, 1]]).astype(np.float32)
    return T_velo_obj, np.linalg.inv(T_velo_obj)


class LidarFrameBuilder(object):
    """One DspgnLidarFrame handle: a camera (K, T_cam_velo, image size) and the loader's config
    (num_lidar_max, min_mask_area, downsample_ratio, read as the reference reads them)."""

    def __init__(self, K, T_cam_velo, configs, img_hw, device=0):
        self.K = np.ascontiguousarray(_np(K), dtype=np.float32).reshape(3, 3)
        self.invK = np.linalg.inv(self.K).astype(np.float32)
        self.T_cam_velo = np.ascontiguousarray(_np(T_cam_velo), dtype=np.float32).reshape(4, 4)
        self.img_h, self.img_w = int(img_hw[0]), int(img_hw[1])
        self.num_lidar_max = int(_cfg_get(configs, "num_lidar_max"))
        self.min_mask_area = int(_cfg_get(configs, "min_mask_area"))
        self.downsample_ratio = int(_cfg_get(configs, "downsample_ratio"))
        self._lib = _lib.load()
        sp = _lib.LidarSpec()
        sp.k[:] = self.K.ravel().tolist()
        sp.inv_k[:] = self.invK.ravel().tolist()
        sp.t_cam_velo[:] = self.T_cam_velo.ravel().tolist()
        sp.img_h, sp.img_w = self.img_h, self.img_w
        sp.num_lidar_max, sp.min_mask_area = self.num_lidar_max, self.min_mask_area
        sp.downsample_ratio = self.downsample_ratio
        h = C.c_void_p()
        _lib.check(self._lib.dspgn_lidar_frame_create(C.byref(sp), int(device), C.byref(h)))
        self._h = h

    def close(self):
        if getattr(self, "_h", None):
            self._lib.dspgn_lidar_frame_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:         # noqa: BLE001 -- interpreter shutdown
            pass

    def set_stream(self, cuda_stream):
        """Enqueue on this cudaStream_t (an int handle; 0 = the legacy default stream) instead of the handle's own."""
        _lib.check(self._lib.dspgn_lidar_frame_set_stream(self._h, C.c_void_p(int(cuda_stream) or None)))

    def detections(self, velo_pts, detections_3d, masks_2d, bboxes_2d):
        """The frame's instances in depth order (kitti_sequence.py:99-216).  velo_pts: (n, 4) float32 as
        load_velo_scan returns it; detections_3d: (k, 7) float32 boxes (x, y, z, w, l, h, theta); masks_2d: (m, H, W)
        bool (an integer mask would mean something else in mask[mask]); bboxes_2d: (m, 4) boxes (l, t, r, b)."""
        velo = np.ascontiguousarray(_np(velo_pts), dtype=np.float32)
        if velo.ndim != 2 or velo.shape[1] != 4:
            raise ValueError("velo_pts must be (n, 4)")
        dets = _np(detections_3d)
        if dets.ndim != 2 or dets.shape[1] < 7:
            raise ValueError("detections_3d must be (k, 7)")
        masks, bboxes = _np(masks_2d), _np(bboxes_2d)
        n_masks = int(masks.shape[0])
        if n_masks:
            if masks.dtype != np.bool_:
                raise TypeError("masks_2d must be bool")
            if masks.shape[1:] != (self.img_h, self.img_w) or bboxes.shape[0] != n_masks:
                raise ValueError("masks_2d must be (m, img_h, img_w) with one bbox per mask")
        dets = dets[np.argsort(dets[:, 0]), :]
        k = dets.shape[0]
        boxes = (_lib.LidarBox * max(k, 1))()
        inst = []
        for n in range(k):
            d = dets[n, :]
            trans, size = d[:3], d[3:6]
            T_velo_obj, T_obj_velo = _box_matrices(d)
            hl = (size / 2)[1]
            hl *= 1.1
            T_cam_obj = self.T_cam_velo @ T_velo_obj
            T_cam_obj[:3, :3] *= hl
            front = T_cam_obj[2, 3] > 0.0
            b = boxes[n]
            b.t_obj_velo[:] = np.asarray(T_obj_velo[:3], np.float32).ravel().tolist()
            b.trans[:] = np.asarray(trans, np.float32).tolist()
            b.size[:] = np.asarray(size, np.float32).tolist()
            b.front = int(bool(front))
            inst.append(ResultDict(T_cam_obj=T_cam_obj, scale=size, is_front=front, rays=None))
        m8 = np.ascontiguousarray(masks).view(np.uint8) if n_masks else None
        bb = np.ascontiguousarray(bboxes[:, :4].astype(np.int32)) if n_masks else None
        out = (_lib.LidarBoxOut * max(k, 1))()
        _lib.check(self._lib.dspgn_lidar_frame_run(
            self._h, velo.ctypes.data_as(_lib._FP), velo.shape[0], boxes, k,
            None if m8 is None else m8.ctypes.data_as(C.POINTER(C.c_uint8)),
            None if bb is None else bb.ctypes.data_as(C.POINTER(C.c_int32)), n_masks, out))
        n_pts = [out[i].n_pts for i in range(k)]
        n_rays = [max(out[i].n_rays, 0) for i in range(k)]
        pts = np.empty((sum(n_pts), 3), np.float32)
        depth = np.empty(sum(n_pts), np.float32)
        rays = np.empty((sum(n_rays), 3), np.float32)
        _lib.check(self._lib.dspgn_lidar_frame_results(self._h, pts.ctypes.data_as(_lib._FP),
                                                      depth.ctypes.data_as(_lib._FP), rays.ctypes.data_as(_lib._FP)))
        p0 = r0 = 0
        for i, it in enumerate(inst):
            it.surface_points = pts[p0:p0 + n_pts[i]]
            it.num_surface_points = n_pts[i]
            if out[i].mask >= 0:
                it.mask = masks[out[i].mask, ...]
                it.bbox = bboxes[out[i].mask, ...]
            if out[i].n_rays >= 0:
                it.rays = rays[r0:r0 + n_rays[i]]
                it.depth = depth[p0:p0 + n_pts[i]]
            p0 += n_pts[i]
            r0 += n_rays[i]
        return inst


def read_calib_file(path):
    """KITTI calib.txt -> {key: float64 array} (the lines up to the first blank one; non-numeric values skipped)."""
    data = {}
    with open(path) as f:
        for line in f:
            if line == "\n":
                break
            key, value = line.split(":", 1)
            try:
                data[key] = np.array([float(x) for x in value.split()])
            except ValueError:
                pass
    return data


def load_velo_scan(path):
    """A velodyne .bin file as (n, 4) float32."""
    return np.fromfile(path, dtype=np.float32).reshape((-1, 4))


class _Frame(object):
    """The loaded frame (the reference's current_frame): id, images, scan and its instances."""

    def __init__(self, frame_id, img_bgr, img_rgb, velo_pts, instances):
        self.frame_id = frame_id
        self.img_bgr, self.img_rgb = img_bgr, img_rgb
        self.img_h, self.img_w = img_rgb.shape[:2]
        self.velo_pts = velo_pts
        self.instances = instances


class KITIISequence(object):
    """Drop-in for reconstruct.kitti_sequence.KITIISequence (kitti_sequence.py:219-260) whose detections are built on
    the device.  Files, calibration and detectors are read as the reference reads them; cv2 is imported on the first
    frame.  Called from C++ with no handler above it (src/Tracking_util.cc:35): get_frame_by_id never raises; a frame
    it cannot build comes back as no detections, with one line on stderr."""

    def __init__(self, data_dir, configs, device=0):
        self.root_dir = data_dir
        self.rgb_dir = os.path.join(data_dir, "image_2")
        self.velo_dir = os.path.join(data_dir, "velodyne")
        self.calib_file = os.path.join(data_dir, "calib.txt")
        self.load_calib()
        self.num_frames = len(os.listdir(self.rgb_dir))
        self.configs = configs
        self.online = _cfg_get(configs, "detect_online")
        self.lbl2d_dir = _cfg_get(configs, "path_label_2d")
        self.lbl3d_dir = _cfg_get(configs, "path_label_3d")
        if not self.online:
            assert self.lbl2d_dir is not None and self.lbl3d_dir is not None
        self.detector_2d, self.detector_3d = None, None
        if self.online:
            from reconstruct import get_detectors
            self.detector_2d, self.detector_3d = get_detectors(configs)
        self.device = device
        self._builder = None
        self.current_frame = None
        self.detections_in_current_frame = None

    def load_calib(self):
        """K and inv(K) of cam2 and T_cam2_velo, float32 (kitti_sequence.py:240-254)."""
        filedata = read_calib_file(self.calib_file)
        P2 = np.reshape(filedata["P2"], (3, 4))
        self.K_cam = P2[0:3, 0:3].astype(np.float32)
        self.invK_cam = np.linalg.inv(self.K_cam).astype(np.float32)
        T_cam0_velo, T_cam2_cam0 = np.eye(4), np.eye(4)
        T_cam0_velo[:3, :] = np.reshape(filedata["Tr"], (3, 4))
        T_cam2_cam0[0, 3] = P2[0, 3] / P2[0, 0]
        self.T_cam_velo = T_cam2_cam0.dot(T_cam0_velo).astype(np.float32)

    def _labels(self, frame_id, img_bgr, velo_file):
        if self.online:
            det_3d = self.detector_3d.make_prediction(velo_file).cpu().numpy()
            det_2d = self.detector_2d.make_prediction(img_bgr)
        else:
            import torch
            det_3d = torch.load(os.path.join(self.lbl3d_dir, "%06d.lbl" % frame_id), weights_only=False)
            det_2d = torch.load(os.path.join(self.lbl2d_dir, "%06d.lbl" % frame_id), weights_only=False)
        return det_3d, det_2d

    def get_frame_by_id(self, frame_id):
        try:
            import cv2
            img_bgr = cv2.imread(os.path.join(self.rgb_dir, "{:06d}".format(frame_id) + ".png"))
            img_rgb = cv2.cvtColor(img_bgr, cv2.COLOR_BGR2RGB)
            velo_file = os.path.join(self.velo_dir, "{:06d}".format(frame_id) + ".bin")
            velo = load_velo_scan(velo_file)
            det_3d, det_2d = self._labels(frame_id, img_bgr, velo_file)
            h, w = img_rgb.shape[:2]
            if self._builder is None or (self._builder.img_h, self._builder.img_w) != (h, w):
                self._builder = LidarFrameBuilder(self.K_cam, self.T_cam_velo, self.configs, (h, w), self.device)
            inst = self._builder.detections(velo, det_3d, det_2d["pred_masks"], det_2d["pred_boxes"])
            self.current_frame = _Frame(frame_id, img_bgr, img_rgb, velo, inst)
        except Exception as e:            # noqa: BLE001 -- see the class comment
            _warn_once(("get_frame_by_id", type(e).__name__), f"get_frame_by_id({frame_id}) failed softly: {e!r}")
            print(f"[dsp_slam_b200] frame {frame_id}: no detections", file=sys.stderr, flush=True)
            inst = []
            self.current_frame = None
        self.detections_in_current_frame = inst
        return inst
