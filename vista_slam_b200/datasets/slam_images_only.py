"""Device-side image preprocessing with the surface of vista_slam/datasets/slam_images_only.py::SLAM_image_only
(SURVEY.md section 8(f) rank 3): `process_image(rgb_image, img_name)` crops, Lanczos-resizes and normalises a frame
exactly like the reference does with PIL + torchvision on the host (bit-exact: tests/test_preprocess.py), but in two
small CUDA kernels, and returns CUDA tensors ready for `_encode_image`.  There is no CPU path."""
import ctypes
import os.path as osp

import numpy as np
import torch

from .. import _lib


class SLAM_image_only:
    def __init__(self, image_paths=(), resolution=(224, 224), device="cuda"):
        if isinstance(resolution, int):
            resolution = (resolution, resolution)
        self.resolution = tuple(int(v) for v in resolution)
        self.color_paths = sorted(image_paths)
        self.n_img = len(self.color_paths)
        self.device = torch.device(device)

    def output_shape(self, H, W, w_edge=10, h_edge=10):
        """(height, width) of the processed frame -- geometry only, no GPU work."""
        hw = (ctypes.c_int * 2)()
        _lib.check(_lib.lib().sta_preprocess_shape(int(H), int(W), self.resolution[0], self.resolution[1], w_edge, h_edge, hw),
                   "sta_preprocess_shape")
        return int(hw[0]), int(hw[1])

    @torch.no_grad()
    def process_image(self, rgb_image, img_name="", w_edge=10, h_edge=10):
        """slam_images_only.py:22-34: HxWx3 uint8 RGB (numpy or torch, host or device) ->
        {'rgb': (3,h,w) fp32 in [-1,1], 'gray': (1,h,w) fp32 in [0,1], 'img_name': basename}, CUDA tensors."""
        if isinstance(rgb_image, np.ndarray):
            rgb_image = torch.from_numpy(np.ascontiguousarray(rgb_image))
        if rgb_image.dtype != torch.uint8 or rgb_image.dim() != 3 or rgb_image.shape[2] != 3:
            raise ValueError("expected an HxWx3 uint8 RGB frame")
        frame = rgb_image.to(self.device, non_blocking=True).contiguous()
        if not frame.is_cuda:
            raise RuntimeError("the CUDA preprocessing has no CPU path")
        H, W, _ = frame.shape
        oh, ow = self.output_shape(H, W, w_edge, h_edge)
        rgb = torch.empty(3, oh, ow, dtype=torch.float32, device=frame.device)
        gray = torch.empty(1, oh, ow, dtype=torch.float32, device=frame.device)
        with torch.cuda.device(frame.device):
            _lib.check(_lib.lib().sta_preprocess_rgb8(_lib.ptr(frame), H, W, self.resolution[0], self.resolution[1], w_edge,
                                                      h_edge, _lib.ptr(rgb), _lib.ptr(gray), None, _lib.cur_stream()),
                       "sta_preprocess_rgb8")
        return {"gray": gray, "rgb": rgb, "img_name": osp.basename(img_name)}

    def __getitem__(self, i):
        """slam_images_only.py:36-40 (run.py:180,193 index the dataset): read frame i from disk as RGB uint8 (cv2 decodes
        BGR; imread_cv2 in vista_slam/utils/image.py converts) and preprocess it on the device."""
        import cv2
        path = self.color_paths[i]
        img = cv2.imread(path, cv2.IMREAD_COLOR)
        if img is None:
            raise IOError("Could not load image=%s" % path)
        return self.process_image(cv2.cvtColor(img, cv2.COLOR_BGR2RGB), osp.basename(path))

    def __len__(self):
        return self.n_img
