"""Device-side segmentation metric (SURVEY.md §8f rank 2): the reference's evaluator moves every image's score map to
the host, takes argmax and builds the confusion matrix with numpy (eval.py:22-29, utils/metric.py:8-33).  Here the
argmax and the confusion matrix are one kernel over the logits that are already in HBM; only classes² + 2 integers
are read back, once per evaluation."""
import ctypes
import math

import numpy as np
import torch

from . import _lib
from ._lib import ptr, stream


def _cv_round(v):
    """cvRound: round half to even (cv2.resize's dsize = saturate_cast<int>(size · f))."""
    return int(np.rint(v))


def image_pre(src_u8, out, *, scaled_hw=None, scale_xy=None, off=(0, 0), mirror_src=False, mirror_out=False, mean, std,
              labels_u8=None, labels_out=None, label_pad=255, clip=None):
    """sigma_image_pre_fwd on one image: src (H0, W0, 3) uint8 CUDA -> out (3, OH, OW) float32 CUDA view (+ labels)."""
    H0, W0, _ = src_u8.shape
    SH, SW = scaled_hw if scaled_hw is not None else (H0, W0)
    sy, sx = scale_xy if scale_xy is not None else (H0 / SH, W0 / SW)
    _, OH, OW = out.shape
    m = (ctypes.c_double * 3)(*[float(v) for v in mean])
    sd = (ctypes.c_double * 3)(*[float(v) for v in std])
    cl = (ctypes.c_int * 4)(*[int(v) for v in clip]) if clip is not None else None
    rc = _lib.lib().sigma_image_pre_fwd(ptr(src_u8), ptr(labels_u8), ptr(out), ptr(labels_out), H0, W0, SH, SW, float(sy), float(sx), OH, OW,
                                        int(off[0]), int(off[1]), int(bool(mirror_src)), int(bool(mirror_out)), int(label_pad), cl, m, sd,
                                        stream())
    _lib.check(rc, "sigma_image_pre_fwd")


class DeviceTrainPre:
    """dataloader/dataloader.py:26-50 (TrainPre) on the device: mirror, random scale, normalize, random crop + pad, for one
    image triple already in HBM as uint8.  The random draws come from `rng` (python `random`-compatible) in the reference's
    order: mirror (random() >= 0.5), scale (choice), crop position (randint per axis, utils/transforms.py:44-59)."""

    def __init__(self, norm_mean, norm_std, image_height, image_width, train_scale_array=None):
        self.mean, self.std = list(norm_mean), list(norm_std)
        self.crop = (int(image_height), int(image_width))
        self.scales = train_scale_array

    def draw(self, h, w, rng):
        mirror = rng.random() >= 0.5
        scale = rng.choice(self.scales) if self.scales is not None else None
        sh, sw = (int(h * scale), int(w * scale)) if scale is not None else (h, w)
        pos_h = rng.randint(0, sh - self.crop[0] + 1) if sh > self.crop[0] else 0
        pos_w = rng.randint(0, sw - self.crop[1] + 1) if sw > self.crop[1] else 0
        return mirror, scale, (pos_h, pos_w)

    def __call__(self, rgb_u8, gt_u8, x_u8, out_rgb, out_gt, out_x, mirror, scale, crop_pos):
        H0, W0, _ = rgb_u8.shape
        sh, sw = (int(H0 * scale), int(W0 * scale)) if scale is not None else (H0, W0)
        ch, cw = self.crop
        # crop rows [y0, y0 + ch) of the scaled image, then centred padding to (ch, cw) (pad_image_to_shape)
        y0, x0 = crop_pos
        got_h, got_w = min(ch, sh - y0), min(cw, sw - x0)
        m_top, m_left = (ch - got_h) // 2, (cw - got_w) // 2
        if got_h < ch and y0 + got_h < sh or got_w < cw and x0 + got_w < sw:
            raise ValueError("crop smaller than the crop size inside the image")   # cannot happen for draw()'s positions
        kw = dict(scaled_hw=(sh, sw), off=(y0 - m_top, x0 - m_left), mirror_src=mirror, mean=self.mean, std=self.std)
        image_pre(rgb_u8, out_rgb, labels_u8=gt_u8, labels_out=out_gt, label_pad=255, **kw)
        image_pre(x_u8, out_x, **kw)


class DeviceEvaluator:
    """engine/evaluator.py:433-522 (sliding_eval_rgbX / scale_process_rgbX / val_func_process_rgbX / process_image_rgbX) with
    everything between the uint8 image and the confusion matrix on the device: multi-scale resize + normalize + pad (+ flip)
    -> batched model forward (all windows of a scale and their flips in ONE batch) -> exp / un-flip / window accumulation ->
    resize back + multi-scale sum (float64) -> argmax -> hist.  Only the uint8 image pair goes up; only the (H, W) uint8
    prediction and classes^2 + 2 integers come down.  The reference's window geometry (x-extents from crop_size[0],
    y-extents from crop_size[1], :472-477) is reproduced as is."""

    def __init__(self, model, num_classes, norm_mean, norm_std, eval_crop_size, eval_stride_rate, multi_scales=(1,), is_flip=False,
                 device="cuda"):
        self.model, self.n = model, int(num_classes)
        self.mean, self.std = [float(v) for v in norm_mean], [float(v) for v in norm_std]
        self.crop = (int(eval_crop_size[0]), int(eval_crop_size[1]))
        self.stride_rate, self.scales, self.flip = float(eval_stride_rate), list(multi_scales), bool(is_flip)
        self.device = torch.device(device)
        self.metric = DeviceMetric(self.n, device=device)

    # -- one scale: returns the scale's score map (ncls, AH, AW) float32 plus the margin / size to resize from
    def _scale(self, rgb_u8, x_u8, s):
        H0, W0, _ = rgb_u8.shape
        same = float(s) == 1.0
        SH, SW = (H0, W0) if same else (_cv_round(H0 * s), _cv_round(W0 * s))
        scale_xy = (1.0, 1.0) if same else (1.0 / s, 1.0 / s)       # cv2.resize(fx=, fy=): scale = 1 / f
        c0, c1 = self.crop
        L_ = _lib.lib()
        if SW <= c1 or SH <= c0:                                       # evaluator.py:458-461: whole image, padded to the crop
            TH, TW = max(SH, c0), max(SW, c1)
            m_top, m_left = (TH - SH) // 2, (TW - SW) // 2
            wins = [(0, 0, SH, SW, -m_top, -m_left, m_top, m_left)]   # (ay, ax, vh, vw, off_y, off_x, tm_top, tm_left)
            AH, AW = SH, SW
        else:                                                          # :462-491 sliding windows
            st0, st1 = int(math.ceil(c0 * self.stride_rate)), int(math.ceil(c1 * self.stride_rate))
            r_grid = int(math.ceil((SH - c0) / st0)) + 1
            c_grid = int(math.ceil((SW - c1) / st1)) + 1
            wh, ww = c1, c0                                            # the reference's extents: rows crop_size[1], cols crop_size[0]
            TH, TW = max(wh, c0), max(ww, c1)
            wins = []
            for gy in range(r_grid):
                for gx in range(c_grid):
                    e_x, e_y = min(gx * st0 + c0, SW), min(gy * st1 + c1, SH)
                    s_x, s_y = e_x - c0, e_y - c1
                    if s_x < 0 or s_y < 0:
                        raise NotImplementedError("window larger than the scaled image (the reference relies on negative numpy slicing here)")
                    tm_top, tm_left = (TH - wh) // 2, (TW - ww) // 2
                    wins.append((s_y, s_x, wh, ww, s_y - tm_top, s_x - tm_left, tm_top, tm_left))
            AH, AW = SH, SW
        nw = len(wins)
        nb = nw * (2 if self.flip else 1)
        rgb = torch.empty((nb, 3, TH, TW), dtype=torch.float32, device=self.device)
        mx = torch.empty_like(rgb)
        for i, (ay, ax, vh, vw, oy, ox, tmt, tml) in enumerate(wins):
            # a window is a crop of the scaled image padded to the tile: pixels outside the WINDOW must be 0 as well
            for src, dst in ((rgb_u8, rgb), (x_u8, mx)):
                self._window(src, dst[i], SH, SW, scale_xy, oy, ox, ay, ax, vh, vw, False)
                if self.flip:
                    self._window(src, dst[nw + i], SH, SW, scale_xy, oy, ox, ay, ax, vh, vw, True)
        with torch.no_grad():
            logits = self.model(rgb, mx).contiguous()
        assert tuple(logits.shape) == (nb, self.n, TH, TW), logits.shape
        acc = torch.zeros((self.n, AH, AW), dtype=torch.float32, device=self.device)
        for i, (ay, ax, vh, vw, oy, ox, tmt, tml) in enumerate(wins):
            lf = logits[nw + i] if self.flip else None
            rc = L_.sigma_eval_exp_accumulate_fwd(ptr(logits[i]), ptr(lf), ptr(acc), self.n, TH, TW, tmt, tml, vh, vw, AH, AW, ay, ax, stream())
            _lib.check(rc, "sigma_eval_exp_accumulate_fwd")
        return acc, SH, SW

    def _window(self, src, dst, SH, SW, scale_xy, oy, ox, ay, ax, vh, vw, mirror_out):
        """One network input: the window [ay, ay+vh) x [ax, ax+vw) of the scaled image, centred in the tile, zeros around."""
        image_pre(src, dst, scaled_hw=(SH, SW), scale_xy=scale_xy, off=(oy, ox), mirror_out=mirror_out, mean=self.mean, std=self.std,
                  clip=(ay, ax, vh, vw))

    def sliding_eval_rgbX(self, img, modal_x, labels=None):
        """img, modal_x: (H, W, 3) uint8 numpy arrays or CUDA tensors -> pred (H, W) uint8 CUDA tensor.  With `labels`
        ((H, W) uint8, 255 = ignore) the running confusion matrix (self.metric) is updated on the device."""
        to = lambda a: a if torch.is_tensor(a) else torch.from_numpy(np.ascontiguousarray(a))
        rgb_u8, x_u8 = to(img).to(self.device, non_blocking=True), to(modal_x).to(self.device, non_blocking=True)
        if rgb_u8.dtype != torch.uint8 or x_u8.dtype != torch.uint8 or rgb_u8.dim() != 3 or rgb_u8.shape[2] != 3 or x_u8.shape != rgb_u8.shape:
            raise ValueError("img / modal_x must be (H, W, 3) uint8 (single-channel modal-x is merged to 3 channels by RGBXDataset)")
        H0, W0, _ = rgb_u8.shape
        total = torch.zeros((H0, W0, self.n), dtype=torch.float64, device=self.device)
        L_ = _lib.lib()
        for s in self.scales:
            acc, SH, SW = self._scale(rgb_u8, x_u8, s)
            rc = L_.sigma_eval_resize_add_fwd(ptr(acc), self.n, acc.shape[1], acc.shape[2], 0, 0, SH, SW, ptr(total), H0, W0, stream())
            _lib.check(rc, "sigma_eval_resize_add_fwd")
        pred = torch.empty((H0, W0), dtype=torch.uint8, device=self.device)
        lab = to(labels).to(self.device) if labels is not None else None
        if lab is not None and (lab.dtype != torch.uint8 or tuple(lab.shape) != (H0, W0)):
            raise ValueError("labels must be (H, W) uint8")
        rc = L_.sigma_eval_argmax_hist_fwd(ptr(total), ptr(lab), ptr(pred), ptr(self.metric.hist), ptr(self.metric.counts), self.n,
                                           H0 * W0, stream())
        _lib.check(rc, "sigma_eval_argmax_hist_fwd")
        return pred


class DeviceMetric:
    """m = DeviceMetric(num_classes); m.update(logits, labels) per batch; hist, labeled, correct = m.result().

    `logits`: (B, classes, H, W) fp32 CUDA tensor; `labels`: (B, H, W) uint8 / int32 / int64 CUDA tensor, pixels whose
    label is outside [0, classes) (255 in the reference's datasets) are ignored — `hist_info`'s `k` mask."""

    def __init__(self, num_classes, device="cuda"):
        self.n = int(num_classes)
        self.hist = torch.zeros(self.n * self.n, dtype=torch.int64, device=device)
        self.counts = torch.zeros(2, dtype=torch.int64, device=device)

    def update(self, logits, labels, pred_out=None):
        if not (logits.is_cuda and labels.is_cuda):
            raise RuntimeError("sigma_b200.DeviceMetric works on CUDA tensors only (there is no CPU path)")
        if logits.dtype != torch.float32:
            raise TypeError("logits must be float32")
        B, C, H, W = logits.shape
        if C != self.n or tuple(labels.shape) != (B, H, W):
            raise ValueError(f"logits {tuple(logits.shape)} / labels {tuple(labels.shape)} do not match {self.n} classes")
        lb = {torch.uint8: 1, torch.int32: 4, torch.int64: 8}.get(labels.dtype)
        if lb is None:
            raise TypeError("labels must be uint8, int32 or int64")
        logits, labels = logits.contiguous(), labels.contiguous()
        pp = pred_out.data_ptr() if pred_out is not None else None
        rc = _lib.lib().sigma_argmax_hist_fwd(logits.data_ptr(), labels.data_ptr(), lb, self.hist.data_ptr(), self.counts.data_ptr(),
                                              pp, B, C, H * W, torch.cuda.current_stream().cuda_stream)
        _lib.check(rc, "sigma_argmax_hist_fwd")

    def result(self):
        h = self.hist.cpu().numpy().reshape(self.n, self.n)
        c = self.counts.cpu().numpy()
        return h, int(c[0]), int(c[1])

    @staticmethod
    def compute_score(hist, correct, labeled):
        """utils/metric.py:17-33: (iou per class, mIoU, freq-weighted IoU, mean class accuracy, pixel accuracy)."""
        hist = np.asarray(hist, dtype=np.float64)
        with np.errstate(divide="ignore", invalid="ignore"):
            iou = np.diag(hist) / (hist.sum(1) + hist.sum(0) - np.diag(hist))
            freq = hist.sum(1) / hist.sum()
            acc = np.diag(hist) / hist.sum(axis=1)
            return iou, float(np.nanmean(iou)), float((iou[freq > 0] * freq[freq > 0]).sum()), float(np.nanmean(acc)), correct / labeled
