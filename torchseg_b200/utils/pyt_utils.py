"""API-compatible helpers (TorchSeg furnace/utils/pyt_utils.py): all_reduce_tensor, load_model,
parse_devices, link_file, ensure_dir, extant_file."""
import argparse
import logging
import os
import time
from collections import OrderedDict

import torch
import torch.distributed as dist

logger = logging.getLogger()


def reduce_tensor(tensor, dst=0, op=dist.ReduceOp.SUM, world_size=1):
    """pyt_utils.py:25-31"""
    out = tensor.clone()
    dist.reduce(out, dst, op)
    if dist.get_rank() == dst:
        out.div_(world_size)
    return out


def all_reduce_tensor(tensor, op=dist.ReduceOp.SUM, world_size=1):
    """pyt_utils.py:34-39: clone → all_reduce(SUM) → / world_size.  Works without an initialised process
    group when world_size == 1 (the reference would raise there)."""
    out = tensor.detach().clone()
    if dist.is_available() and dist.is_initialized():
        dist.all_reduce(out, op)
    out.div_(world_size)
    return out


def load_model(model, model_file, is_restore=False):
    """pyt_utils.py:42-79: non-strict load with missing / unexpected key logging; `is_restore` re-adds the
    'module.' prefix that Engine.save_checkpoint strips."""
    t0 = time.time()
    if isinstance(model_file, str):
        state_dict = torch.load(model_file, map_location=torch.device('cpu'))
        if 'model' in state_dict.keys():
            state_dict = state_dict['model']
    else:
        state_dict = model_file
    t1 = time.time()
    if is_restore:
        state_dict = OrderedDict(('module.' + k, v) for k, v in state_dict.items())
    model.load_state_dict(state_dict, strict=False)
    ckpt_keys, own_keys = set(state_dict.keys()), set(model.state_dict().keys())
    missing, unexpected = own_keys - ckpt_keys, ckpt_keys - own_keys
    if missing:
        logger.warning('Missing key(s) in state_dict: {}'.format(', '.join(sorted(missing))))
    if unexpected:
        logger.warning('Unexpected key(s) in state_dict: {}'.format(', '.join(sorted(unexpected))))
    logger.info("Load model, Time usage:\n\tIO: {}, initialize parameters: {}".format(t1 - t0, time.time() - t1))
    return model


def parse_devices(input_devices):
    """pyt_utils.py:82-106 ('0', '0,1', '0-3', '*'); an empty string means "no explicit device list" (CPU or the
    current CUDA device) instead of the reference's ValueError (SURVEY.md App. C4)."""
    n = torch.cuda.device_count()
    if input_devices is None or input_devices == '':
        return list(range(n)) if n > 0 else [0]
    if input_devices.endswith('*'):
        return list(range(n)) if n > 0 else [0]
    devices = []
    for d in input_devices.split(','):
        if '-' in d:
            a, b = d.split('-')[0], d.split('-')[1]
            assert a != '' and b != ''
            a, b = int(a), int(b)
            assert a < b and b < max(n, 1)
            devices.extend(range(a, b + 1))
        else:
            dev = int(d)
            assert dev < max(n, 1)
            devices.append(dev)
    logger.info('using devices {}'.format(', '.join(str(d) for d in devices)))
    return devices


def extant_file(x):
    """argparse type: path must exist (pyt_utils.py:109-117)"""
    if not os.path.exists(x):
        raise argparse.ArgumentTypeError("{0} does not exist".format(x))
    return x


def link_file(src, target):
    """pyt_utils.py:120-123 (os.symlink instead of shelling out to `ln -s`)"""
    if os.path.isdir(target) or os.path.isfile(target) or os.path.islink(target):
        os.remove(target)
    os.symlink(src, target)


def ensure_dir(path):
    if not os.path.isdir(path):
        os.makedirs(path)
