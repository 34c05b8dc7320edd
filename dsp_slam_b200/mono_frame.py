"""A monocular (Redwood / Freiburg) keyframe's object detection built on the H100 (libdspgn's DspgnMonoFrame).

    MonoFrameBuilder(K, k1, k2, configs, img_hw, mask_erosion).detections(masks_2d, bboxes_2d, keypoints=None)
    MonoSequence(data_dir, configs).get_frame_by_id(frame_id)          reconstruct/mono_sequence.py:117-153

`detections` returns the instance list of the reference's Frame.get_detections (reconstruct/mono_sequence.py:75-114)
bit for bit: [] without masks, else one ResultDict for the largest mask with bbox (a view of the chosen row), mask
(masks_2d[i].astype(float32) * 255., built on the host from the index the device returns) and background_rays.  The
background sampler, the undistortion (cv2.undistortPoints restated) and the rays run on the device in one call, which
also tests the keyframe's keypoints against the mask eroded by Objects.maskErrosion, as Tracking::
GetObjectDetectionsMono does (src/Tracking_util.cc:176-201) without eroding the image: `feature_points()` returns
their indices.  A frame the reference fails on (fewer than 2 background pixels) raises ValueError here.
"""
import ctypes as C
import os
import sys

import numpy as np

from . import _lib
from .lidar_frame import _np
from .optimizer import ResultDict, _cfg_get, _cfg_has, _warn_once


class MonoFrameBuilder(object):
    """One DspgnMonoFrame handle: a camera (K and inv(K) float64, k1, k2, image size), the loader's downsample_ratio
    and the Tracking yaml's Objects.maskErrosion (mask_erosion=None: configs' mask_erosion if present, else 0)."""

    def __init__(self, K, k1, k2, configs, img_hw, mask_erosion=None, device=0):
        self.K = np.ascontiguousarray(_np(K), dtype=np.float64).reshape(3, 3)
        self.invK = np.linalg.inv(self.K)
        self.k1, self.k2 = float(k1), float(k2)
        self.img_h, self.img_w = int(img_hw[0]), int(img_hw[1])
        self.downsample_ratio = int(_cfg_get(configs, "downsample_ratio"))
        if mask_erosion is None:
            mask_erosion = _cfg_get(configs, "mask_erosion") if _cfg_has(configs, "mask_erosion") else 0
        self.mask_erosion = int(mask_erosion)
        self._lib = _lib.load()
        sp = _lib.MonoSpec()
        sp.k[:] = self.K.ravel().tolist()
        sp.inv_k[:] = self.invK.ravel().tolist()
        sp.k1, sp.k2 = self.k1, self.k2
        sp.img_h, sp.img_w = self.img_h, self.img_w
        sp.downsample_ratio, sp.mask_erosion = self.downsample_ratio, self.mask_erosion
        h = C.c_void_p()
        _lib.check(self._lib.dspgn_mono_frame_create(C.byref(sp), int(device), C.byref(h)))
        self._h = h
        self._features = np.zeros(0, np.int32)
        self.last = None

    def close(self):
        if getattr(self, "_h", None):
            self._lib.dspgn_mono_frame_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:         # noqa: BLE001 -- interpreter shutdown
            pass

    def set_stream(self, cuda_stream):
        """Enqueue on this cudaStream_t (an int handle; 0 = the legacy default stream) instead of the handle's own."""
        _lib.check(self._lib.dspgn_mono_frame_set_stream(self._h, C.c_void_p(int(cuda_stream) or None)))

    def detections(self, masks_2d, bboxes_2d, keypoints=None):
        """The frame's instances (mono_sequence.py:86-114).  masks_2d: (m, H, W) bool; bboxes_2d: (m, 4) boxes
        (l, t, r, b); keypoints: None or (n, 2) float32 (pt.x, pt.y) for feature_points()."""
        masks, bboxes = _np(masks_2d), _np(bboxes_2d)
        n_masks = int(masks.shape[0])
        if n_masks:
            if masks.dtype != np.bool_:
                raise TypeError("masks_2d must be bool")
            if masks.shape[1:] != (self.img_h, self.img_w) or bboxes.shape[0] != n_masks:
                raise ValueError("masks_2d must be (m, img_h, img_w) with one bbox per mask")
        kp = np.zeros((0, 2), np.float32) if keypoints is None else \
            np.ascontiguousarray(_np(keypoints), dtype=np.float32).reshape(-1, 2)
        m8 = np.ascontiguousarray(masks).view(np.uint8) if n_masks else None
        bb = np.ascontiguousarray(bboxes[:, :4].astype(np.int32)) if n_masks else None
        out = _lib.MonoOut()
        _lib.check(self._lib.dspgn_mono_frame_run(
            self._h, None if m8 is None else m8.ctypes.data_as(C.POINTER(C.c_uint8)),
            None if bb is None else bb.ctypes.data_as(C.POINTER(C.c_int32)), n_masks,
            kp.ctypes.data_as(_lib._FP), kp.shape[0], C.byref(out)))
        self.last = out
        rays = np.empty((max(out.n_rays, 0), 3), np.float32)
        feats = np.empty(out.n_feature, np.int32)
        _lib.check(self._lib.dspgn_mono_frame_results(self._h, rays.ctypes.data_as(_lib._FP),
                                                     feats.ctypes.data_as(C.POINTER(C.c_int32))))
        self._features = feats
        if out.mask < 0:
            return []
        if out.n_rays < 0:
            raise ValueError(f"{out.n_nonsurface} background pixel(s) in the largest mask's bbox: the reference "
                             "cannot undistort fewer than 2")
        return [ResultDict(bbox=bboxes[out.mask, ...], mask=masks[out.mask, ...].astype(np.float32) * 255.,
                           background_rays=rays)]

    def feature_points(self):
        """Ascending int32 indices of the last call's keypoints inside the eroded largest mask (the detection is good
        iff there are at least 20)."""
        return self._features


class _Frame(object):
    """The loaded frame (the reference's current_frame): id, images and its instances."""

    def __init__(self, frame_id, img_bgr, img_rgb, instances):
        self.frame_id = frame_id
        self.img_bgr, self.img_rgb = img_bgr, img_rgb
        self.img_h, self.img_w = img_rgb.shape[:2]
        self.instances = instances


class MonoSequence(object):
    """Drop-in for reconstruct.mono_sequence.MonoSequence (mono_sequence.py:117-153) whose detection is built on the
    device.  The yaml, the images, the stored labels and the online detector are read as the reference reads them.
    Called from C++ with no handler above it (src/Tracking_util.cc:166): get_frame_by_id never raises; a frame it
    cannot build (including the reference's failures on fewer than 2 background pixels) comes back as no instances,
    with one line on stderr."""

    def __init__(self, data_dir, configs, device=0):
        import cv2
        self.root_dir = data_dir
        self.rgb_dir = os.path.join(data_dir, "image_0")
        fs = cv2.FileStorage(_cfg_get(configs, "slam_config_path"), cv2.FILE_STORAGE_READ)
        fx, fy = fs.getNode("Camera.fx").real(), fs.getNode("Camera.fy").real()
        cx, cy = fs.getNode("Camera.cx").real(), fs.getNode("Camera.cy").real()
        self.k1, self.k2 = fs.getNode("Camera.k1").real(), fs.getNode("Camera.k2").real()
        erosion = fs.getNode("Objects.maskErrosion")
        self.mask_erosion = 0 if erosion.empty() else int(erosion.real())
        self.K_cam = np.array([[fx, 0.0, cx], [0.0, fy, cy], [0.0, 0.0, 1.0]])
        self.invK_cam = np.linalg.inv(self.K_cam)
        self.configs = configs
        self.data_type = _cfg_get(configs, "data_type")
        assert self.data_type in ("Redwood", "Freiburg"), "Wrong data type, supported: Redwood and Freiburg"
        self.online = _cfg_get(configs, "detect_online")
        self.lbl2d_dir = _cfg_get(configs, "path_label_2d") if _cfg_has(configs, "path_label_2d") else None
        if not self.online:
            assert self.lbl2d_dir is not None
        self.detector_2d = None
        if self.online:
            from reconstruct import get_detectors
            self.detector_2d = get_detectors(configs)
        self.device = device
        self._builder = None
        self.current_frame = None
        self.detections_in_current_frame = None

    def _labels(self, frame_id, img_bgr):
        if self.online:
            cls = "chairs" if self.data_type == "Redwood" else "cars"
            return self.detector_2d.make_prediction(img_bgr, object_class=cls)
        import torch
        return torch.load(os.path.join(self.lbl2d_dir, "%06d.lbl" % frame_id), weights_only=False)

    def get_frame_by_id(self, frame_id):
        try:
            import cv2
            img_bgr = cv2.imread(os.path.join(self.rgb_dir, "{:06d}".format(frame_id) + ".png"))
            img_rgb = cv2.cvtColor(img_bgr, cv2.COLOR_BGR2RGB)
            det_2d = self._labels(frame_id, img_bgr)
            h, w = img_rgb.shape[:2]
            if self._builder is None or (self._builder.img_h, self._builder.img_w) != (h, w):
                self._builder = MonoFrameBuilder(self.K_cam, self.k1, self.k2, self.configs, (h, w),
                                                 self.mask_erosion, self.device)
            inst = self._builder.detections(det_2d["pred_masks"], det_2d["pred_boxes"])
            self.current_frame = _Frame(frame_id, img_bgr, img_rgb, inst)
        except Exception as e:            # noqa: BLE001 -- see the class comment
            _warn_once(("get_frame_by_id", type(e).__name__), f"get_frame_by_id({frame_id}) failed softly: {e!r}")
            print(f"[dsp_slam_b200] frame {frame_id}: no detections", file=sys.stderr, flush=True)
            inst = []
            self.current_frame = None
        self.detections_in_current_frame = inst
        return inst
