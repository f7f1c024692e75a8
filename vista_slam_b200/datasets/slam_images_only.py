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

    @torch.no_grad()
    def process_images(self, rgb_frames, img_names=None, w_edge=10, h_edge=10):
        """process_image over F same-size HxWx3 uint8 RGB frames (a list, or an (F, H, W, 3) array or tensor) in one
        launch pair -> {'rgb': (F,3,h,w), 'gray': (F,1,h,w), 'img_name': [basenames]}, CUDA tensors, every frame
        bit-identical to its own process_image.  rgb[i:i+1] and gray[i] are what step_many and compute_disparity
        take; gray feeds FlowTracker.compute_disparities as it is."""
        if isinstance(rgb_frames, (np.ndarray, torch.Tensor)):
            frames = [rgb_frames[i] for i in range(rgb_frames.shape[0])] if rgb_frames.ndim == 4 else None
        else:
            frames = list(rgb_frames)
        if frames is None or any(not isinstance(f, (np.ndarray, torch.Tensor)) or f.ndim != 3 or f.shape[2] != 3
                                 or f.dtype not in (np.uint8, torch.uint8) for f in frames):
            raise ValueError("expected HxWx3 uint8 RGB frames")
        F = len(frames)
        if F and len({tuple(f.shape) for f in frames}) > 1:
            raise ValueError("all frames must have the same size")
        names = [""] * F if img_names is None else [osp.basename(n) for n in img_names]
        if len(names) != F:
            raise ValueError("one image name per frame")
        if F == 0:
            raise ValueError("no frames")
        H, W, _ = frames[0].shape
        oh, ow = self.output_shape(H, W, w_edge, h_edge)
        if isinstance(rgb_frames, (np.ndarray, torch.Tensor)):
            batch = torch.as_tensor(rgb_frames)
        elif all(isinstance(f, np.ndarray) for f in frames):
            batch = torch.from_numpy(np.stack(frames))
        else:
            batch = torch.stack([torch.as_tensor(f).to(self.device) for f in frames])
        batch = batch.to(self.device, non_blocking=True).contiguous()
        if not batch.is_cuda:
            raise RuntimeError("the CUDA preprocessing has no CPU path")
        rgb = torch.empty(F, 3, oh, ow, dtype=torch.float32, device=batch.device)
        gray = torch.empty(F, 1, oh, ow, dtype=torch.float32, device=batch.device)
        with torch.cuda.device(batch.device):
            _lib.check(_lib.lib().sta_preprocess_rgb8_many(_lib.ptr(batch), F, H, W, self.resolution[0], self.resolution[1],
                                                           w_edge, h_edge, _lib.ptr(rgb), _lib.ptr(gray), None,
                                                           _lib.cur_stream()), "sta_preprocess_rgb8_many")
        return {"gray": gray, "rgb": rgb, "img_name": names}

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
