"""Evaluator with the reference's surface (TorchSeg furnace/engine/evaluator.py): `whole_eval`, `sliding_eval`,
`scale_process`, `val_func_process`, `process_image`, `func_per_iteration` / `compute_metric` hooks and a
single-process `run`. SURVEY.md §8f rank 2 — the first slice of the evaluator row.

What is GPU-first here: all sliding-window crops of one scale go through the network in ONE batched forward (the
reference runs them one by one, evaluator.py:222-239) and are accumulated on the device; the eval-mode network forward
itself is the libtsb path (BN from running statistics). What deliberately stays on the host, exactly like the
reference, so that predictions can be compared pixel by pixel: cv2 resizing of the input per scale and of the
accumulated score map back to the original size. Quirks kept: overlapping windows are SUMMED, not averaged
(`score = data_scale`, evaluator.py:241-242); flipped scores are added before `exp` is taken.

`sliding_eval_device` / `whole_eval_device` run all of that on the device instead (libtsb tsb_eval_windows,
tsb_eval_accumulate, tsb_eval_resize_add): the uint8 frame is uploaded once, and the int64 prediction they return is
identical, pixel for pixel, to what `sliding_eval` / `whole_eval` return for the same `val_func` (fp32 log-probs; image
mean / std as float64, like the configs). Pair them with `metric.hist_info_torch` so that only the n_cl² confusion counts
come back to the host.

`multi_process_evaluation` / `worker` (evaluator.py:97-163): one spawned process per device, the dataset split in
contiguous shreds, results returned through a queue; `run` uses it when more than one device is given. Not carried over:
datasets / visualisation helpers."""
import os
import time

import numpy as np
import torch

from .logger import get_logger
from .. import ops
from ..utils.gpu_pipeline import normalize_lut
from ..utils.img_utils import get_2dshape, normalize, pad_image_to_shape
from ..utils.pyt_utils import ensure_dir, link_file, load_model

logger = get_logger()


class Evaluator(object):
    def __init__(self, dataset, class_num, image_mean, image_std, network, multi_scales, is_flip, devices, verbose=False,
                 save_path=None, show_image=False, crop_batch=8):
        self.dataset = dataset
        self.ndata = self.dataset.get_length() if dataset is not None else 0
        self.class_num = class_num
        self.image_mean = image_mean
        self.image_std = image_std
        self.multi_scales = multi_scales
        self.is_flip = is_flip
        self.network = network
        self.devices = devices
        self.val_func = None
        self.verbose = verbose
        self.save_path = save_path
        if save_path is not None:
            ensure_dir(save_path)
        self.show_image = show_image
        self.crop_batch = crop_batch     # windows per batched forward
        self.context = None              # torch.multiprocessing 'spawn' context, created on first use (evaluator.py:36-37)
        self.results_queue = None

    # ------------------------------------------------------------------ driver (evaluator.py:43-95)
    def run(self, model_path, model_indice, log_file, log_file_link):
        """-e x.pth | -e epoch | -e start-end | -e start-  (same four modes as the reference)"""
        if '.pth' in model_indice:
            models = [model_indice]
        elif "-" in model_indice:
            start = int(model_indice.split("-")[0])
            end = model_indice.split("-")[1]
            names = [m for m in os.listdir(model_path) if m != "epoch-last.pth"]
            idx = sorted(int(m.split(".")[0].split("-")[1]) for m in names)
            if end:
                idx = [i for i in idx if start <= i <= int(end)]
            else:
                idx = [i for i in idx if i >= start]
            models = [os.path.join(model_path, "epoch-%d.pth" % i) for i in idx]
        else:
            models = [os.path.join(model_path, 'epoch-%s.pth' % model_indice)]
        results = open(log_file, 'a')
        link_file(log_file, log_file_link)
        for model in models:
            logger.info("Load Model: %s" % model)
            self.val_func = load_model(self.network, model)
            result_line = (self.multi_process_evaluation() if len(self.devices) > 1 else self.single_process_evalutation())
            results.write('Model: ' + model + '\n')
            results.write(result_line)
            results.write('\n')
            results.flush()
        results.close()

    def single_process_evalutation(self):
        """evaluator.py:84-95 (the reference's spelling of the method name is part of its API)"""
        t0 = time.perf_counter()
        logger.info('GPU %s handle %d data.' % (self.devices[0], self.ndata))
        all_results = [self.func_per_iteration(self.dataset[idx], self.devices[0]) for idx in range(self.ndata)]
        result_line = self.compute_metric(all_results)
        logger.info('Evaluation Elapsed Time: %.2fs' % (time.perf_counter() - t0))
        return result_line

    def multi_process_evaluation(self):
        """evaluator.py:97-146: one process per device over contiguous shreds of the dataset, results through a queue"""
        import torch.multiprocessing as mp
        t0 = time.perf_counter()
        if self.context is None:
            self.context = mp.get_context('spawn')
        self.results_queue = self.context.Queue(max(1, self.ndata))
        nr_devices = len(self.devices)
        stride = int(np.ceil(self.ndata / nr_devices))
        shreds = [list(range(d * stride, min((d + 1) * stride, self.ndata))) for d in range(nr_devices)]
        all_results = []
        if nr_devices > 1:
            procs = []
            for d, device in enumerate(self.devices):
                logger.info('GPU %s handle %d data.' % (device, len(shreds[d])))
                procs.append(self.context.Process(target=self.worker, args=(shreds[d], device)))
            for p in procs:
                p.start()
            for _ in range(self.ndata):
                all_results.append(self.results_queue.get())
                if self.verbose:
                    self.compute_metric(all_results)
            for p in procs:
                p.join()
        else:
            self.worker(shreds[0], self.devices[0])
            for _ in range(self.ndata):
                all_results.append(self.results_queue.get())
        result_line = self.compute_metric(all_results)
        logger.info('Evaluation Elapsed Time: %.2fs' % (time.perf_counter() - t0))
        return result_line

    def worker(self, shred_list, device):
        """evaluator.py:148-163"""
        t0 = time.time()
        logger.info('Load Model on Device %s: %.2fs' % (device, time.time() - t0))
        for idx in shred_list:
            results_dict = self.func_per_iteration(self.dataset[idx], device)
            self.results_queue.put(results_dict)

    def __getstate__(self):
        state = dict(self.__dict__)
        state['context'] = None          # a multiprocessing context is not picklable; the queue travels as a Process argument owner
        return state

    def func_per_iteration(self, data, device):
        raise NotImplementedError

    def compute_metric(self, results):
        raise NotImplementedError

    # ------------------------------------------------------------------ evaluation of one image
    def whole_eval(self, img, output_size, input_size=None, device=None):
        """evaluator.py:163-182: one forward over the (optionally padded) image"""
        import cv2
        margin = None
        if input_size is not None:
            img, margin = self.process_image(img, input_size)
        else:
            img = self.process_image(img, input_size)
        pred = self.val_func_process(img, device)
        if margin is not None:
            pred = pred[:, margin[0]:(pred.shape[1] - margin[1]), margin[2]:(pred.shape[2] - margin[3])]
        pred = pred.permute(1, 2, 0).cpu().numpy()
        if output_size is not None:
            pred = cv2.resize(pred, (output_size[1], output_size[0]), interpolation=cv2.INTER_LINEAR)
        return pred.argmax(2)

    def sliding_eval(self, img, crop_size, stride_rate, device=None):
        """evaluator.py:185-199: sum of the per-scale score maps, argmax"""
        import cv2
        rows, cols, _ = img.shape
        total = np.zeros((rows, cols, self.class_num))
        for s in self.multi_scales:
            scaled = cv2.resize(img, None, fx=s, fy=s, interpolation=cv2.INTER_LINEAR)
            total += self.scale_process(scaled, (rows, cols), crop_size, stride_rate, device)
        return total.argmax(2)

    def window_grid(self, pad_rows, pad_cols, crop_size, stride_rate):
        """top-left corners of the sliding windows in the reference's raster order (evaluator.py:215-231)"""
        stride = int(np.ceil(crop_size * stride_rate))
        r_grid = int(np.ceil((pad_rows - crop_size) / stride)) + 1
        c_grid = int(np.ceil((pad_cols - crop_size) / stride)) + 1
        corners = []
        for gy in range(r_grid):
            for gx in range(c_grid):
                e_x = min(gx * stride + crop_size, pad_cols)
                e_y = min(gy * stride + crop_size, pad_rows)
                corners.append((e_y - crop_size, e_x - crop_size))
        return corners

    def scale_process(self, img, ori_shape, crop_size, stride_rate, device=None):
        """evaluator.py:201-251 with the windows batched through the network"""
        import cv2
        new_rows, new_cols, _ = img.shape
        if max(new_rows, new_cols) <= crop_size:
            input_data, margin = self.process_image(img, crop_size)
            score = self.val_func_process(input_data, device)
            score = score[:, margin[0]:(score.shape[1] - margin[1]), margin[2]:(score.shape[2] - margin[3])]
        else:
            img_pad, margin = pad_image_to_shape(img, crop_size, cv2.BORDER_CONSTANT, value=0)
            pad_rows, pad_cols = img_pad.shape[:2]
            corners = self.window_grid(pad_rows, pad_cols, crop_size, stride_rate)
            norm = self.process_image(img_pad)          # normalise once; every window is a crop of it ([3, H, W])
            data_scale = None
            for b0 in range(0, len(corners), self.crop_batch):
                chunk = corners[b0:b0 + self.crop_batch]
                batch = np.stack([norm[:, y:y + crop_size, x:x + crop_size] for y, x in chunk])
                scores = self.val_func_process(batch, device, batched=True)        # [n, class, crop, crop] on the device
                if data_scale is None:
                    data_scale = torch.zeros((self.class_num, pad_rows, pad_cols), dtype=scores.dtype, device=scores.device)
                for (y, x), sc in zip(chunk, scores):   # windows are SUMMED, not averaged (evaluator.py:241-242)
                    data_scale[:, y:y + crop_size, x:x + crop_size] += sc
            score = data_scale[:, margin[0]:(data_scale.shape[1] - margin[1]), margin[2]:(data_scale.shape[2] - margin[3])]
        score = score.permute(1, 2, 0).cpu().numpy()
        return cv2.resize(score, (ori_shape[1], ori_shape[0]), interpolation=cv2.INTER_LINEAR)

    # ------------------------------------------------------------------ the same evaluation on the device
    def sliding_eval_device(self, img, crop_size, stride_rate, device):
        """sliding_eval with the resizes, windows, score sums and arg-max on the device: uint8 [rows, cols, 3] numpy frame →
        int64 [rows, cols] device tensor, equal to sliding_eval(img, crop_size, stride_rate, device)"""
        dev = _cuda_device(device)
        src = torch.from_numpy(np.ascontiguousarray(img)).to(dev)
        rows, cols = img.shape[:2]
        total = torch.zeros((self.class_num, rows, cols), dtype=torch.float64, device=dev)     # sum over scales
        pred = torch.zeros((rows, cols), dtype=torch.int64, device=dev)
        for i, s in enumerate(self.multi_scales):
            score = self._scale_process_device(src, s, crop_size, stride_rate, dev)
            ops.eval_resize_add(score, total, pred if i == len(self.multi_scales) - 1 else None)
        return pred

    def whole_eval_device(self, img, output_size, input_size=None, device=None):
        """whole_eval on the device: uint8 [rows, cols, 1 | 3] numpy frame → int64 device tensor of size output_size (or
        the frame's), equal to whole_eval(img, output_size, input_size, device)"""
        dev = _cuda_device(device)
        src = torch.from_numpy(np.ascontiguousarray(img)).to(dev)
        rows, cols = img.shape[:2]
        th, tw = get_2dshape(input_size) if input_size is not None else (rows, cols)
        win = (max(th, rows), max(tw, cols))                      # one window: the whole padded image
        score = self._canvas_scores(src, None, rows, cols, (th, tw), True, [(0, 0)], win, dev, None)
        out_h, out_w = (int(output_size[0]), int(output_size[1])) if output_size is not None else (rows, cols)
        total = torch.zeros((score.shape[0], out_h, out_w), dtype=torch.float64, device=dev)
        pred = torch.empty((out_h, out_w), dtype=torch.int64, device=dev)
        ops.eval_resize_add(score, total, pred)
        return pred

    def _scale_process_device(self, src, s, crop_size, stride_rate, dev):
        """scale_process for one scale: the margin-cropped [class, h, w] fp32 score view of the scaled frame. One window
        (max side <= crop) pads the normalised image with 0.0, the sliding branch the uint8 image with 0."""
        rows, cols = src.shape[:2]
        sh, sw = int(round(rows * s)), int(round(cols * s))      # cv2's dsize for fx = fy = s (round half to even)
        corners = self.window_grid(max(sh, crop_size), max(sw, crop_size), crop_size, stride_rate)
        return self._canvas_scores(src, s, sh, sw, (crop_size, crop_size), max(sh, sw) <= crop_size, corners,
                                   (crop_size, crop_size), dev, self.class_num)

    def _canvas_scores(self, src, fx, sh, sw, pad_shape, pad_zero, corners, win, dev, class_num):
        """the frame scaled by fx to (sh, sw), padded up to pad_shape (pad_image_to_shape's margins), cut into win-sized
        windows at `corners`, crop_batch per forward, their scores summed on the canvas; returns the margin-cropped view"""
        PH, PW = max(pad_shape[0], sh), max(pad_shape[1], sw)
        ph, pw = PH - sh, PW - sw
        m = (ph // 2, ph - ph // 2, pw // 2, pw - pw // 2)
        wh, ww = win
        lut = torch.from_numpy(normalize_lut(self.image_mean, self.image_std)).to(dev)
        acc = None
        for b0 in range(0, len(corners), self.crop_batch):
            chunk = torch.tensor(corners[b0:b0 + self.crop_batch], dtype=torch.int32).to(dev)
            x = ops.eval_windows(src, fx, sh, sw, m[0], m[2], lut, pad_zero, chunk, wh, ww)
            xf = ops.eval_windows(src, fx, sh, sw, m[0], m[2], lut, pad_zero, chunk, wh, ww, mirror=True) if self.is_flip else None
            lp, lpf = self._log_probs(x, xf, dev)
            if acc is None:
                C = lp.shape[1]
                if class_num is not None and C != class_num:
                    raise ValueError("val_func returns %d classes, the evaluator expects %d" % (C, class_num))
                acc = torch.zeros((C, PH, PW), dtype=torch.float32, device=dev)
            ops.eval_accumulate(lp, lpf, chunk, acc)
        return acc[:, m[0]:PH - m[1], m[2]:PW - m[3]]

    def _log_probs(self, x, xf, dev):
        """the network calls of val_func_process (same module state, same order): log-probs of the windows and of the
        mirrored windows, as contiguous fp32"""
        self.val_func.eval()
        if hasattr(self.val_func, "to"):
            self.val_func.to(dev)
        with torch.no_grad():
            out = [self.val_func(x)] + ([self.val_func(xf)] if xf is not None else [])
        for t in out:
            if t.dtype != torch.float32:
                raise TypeError("the device evaluator sums fp32 log-probs; val_func returned %s" % t.dtype)
        out = [t.contiguous() for t in out]
        return out[0], (out[1] if xf is not None else None)

    def val_func_process(self, input_data, device=None, batched=False):
        """evaluator.py:253-273: exp(log-prob(x) [+ flip(log-prob(flip(x)))]); returns [class, h, w] (or [n, class, h, w])"""
        arr = np.ascontiguousarray(input_data if batched else input_data[None], dtype=np.float32)
        x = torch.as_tensor(arr)
        if device is not None:
            x = x.to(device, non_blocking=True)
        self.val_func.eval()
        if device is not None and hasattr(self.val_func, "to"):
            self.val_func.to(device)
        with torch.no_grad():
            score = self.val_func(x)
            if self.is_flip:
                score = score + self.val_func(x.flip(-1)).flip(-1)
            score = torch.exp(score.float())
        return score if batched else score[0]

    def process_image(self, img, crop_size=None):
        """evaluator.py:275-297: grey → 3 channels, normalise, optional centred zero padding, HWC → CHW"""
        import cv2
        p_img = img
        if img.shape[2] < 3:
            p_img = np.concatenate((p_img, p_img, p_img), axis=2)
        p_img = normalize(p_img, self.image_mean, self.image_std)
        if crop_size is not None:
            p_img, margin = pad_image_to_shape(p_img, crop_size, cv2.BORDER_CONSTANT, value=0)
            return p_img.transpose(2, 0, 1), margin
        return p_img.transpose(2, 0, 1)


def _cuda_device(device):
    """the CUDA device of the device evaluator (None: the current one)"""
    if device is None:
        return torch.device("cuda", torch.cuda.current_device())
    dev = torch.device("cuda", device) if isinstance(device, int) else torch.device(device)
    if dev.type != "cuda":
        raise ValueError("the device evaluator runs on a CUDA device, got %s" % dev)
    return dev
