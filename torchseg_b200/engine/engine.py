"""Engine / State with the reference API (TorchSeg furnace/engine/engine.py:23-163): argparse injection
(-d / -c / --local_rank), WORLD_SIZE detection, process-group init, state registry, checkpoint
save / link / restore in the reference's on-disk format.

Differences (documented in INTEGRATION.md): the backend is NCCL when CUDA is present and gloo otherwise
(CPU tests), LOCAL_RANK from the environment is honoured (torchrun), `-d ''` no longer raises, and a
world of one process under torchrun still counts as "distributed" when TSB_FORCE_DISTRIBUTED=1.
"""
import argparse
import os
import os.path as osp
import time
from collections import OrderedDict

import torch
import torch.distributed as dist

from .logger import get_logger
from .version import __version__
from ..utils.pyt_utils import load_model, parse_devices, extant_file, link_file, ensure_dir

logger = get_logger()


_STATE_FIELDS = ('epoch', 'iteration', 'dataloader', 'model', 'optimizer')


class State(object):
    """training-state registry (engine.py:23-35): epoch / iteration counters plus the objects a checkpoint needs"""

    def __init__(self):
        for name in _STATE_FIELDS:
            setattr(self, name, 0 if name in ('epoch', 'iteration') else None)

    def register(self, **kwargs):
        unknown = [k for k in kwargs if k not in _STATE_FIELDS]
        if unknown:
            raise AssertionError("unknown state field(s): %s" % ", ".join(unknown))
        self.__dict__.update(kwargs)


def _portable_state_dict(model):
    """model.state_dict() in the on-disk convention of engine.py:94-106: no DistributedDataParallel `module.` prefix,
    plain contiguous CPU tensors (NCHW fp32 whatever the in-memory KRSC layout)"""
    out = OrderedDict()
    for key, value in model.state_dict().items():
        if key.startswith('module.'):
            key = key[len('module.'):]
        out[key] = value.detach().contiguous().cpu() if torch.is_tensor(value) else value
    return out


class Engine(object):
    """context manager around a training script (engine.py:38-163): CLI, process group, state, checkpoints"""

    def __init__(self, custom_parser=None, argv=None):
        self.version = __version__
        logger.info("PyTorch Version {}, Furnace(libtsb) Version {}".format(torch.__version__, self.version))
        self.state = State()
        self.devices, self.distributed, self.local_rank, self.world_size = None, False, 0, 1
        if custom_parser is not None and not isinstance(custom_parser, argparse.ArgumentParser):
            raise AssertionError("custom_parser must be an argparse.ArgumentParser")
        self.parser = custom_parser if custom_parser is not None else argparse.ArgumentParser()
        self.inject_default_parser()
        self.args = self.parser.parse_args(argv)
        self.continue_state_object = self.args.continue_fpath
        self._setup_world()

    def _setup_world(self):
        """WORLD_SIZE in the environment (torch.distributed launchers) → one process per GPU; otherwise the -d list"""
        world = os.environ.get('WORLD_SIZE')
        if world is not None:
            self.distributed = int(world) > 1 or os.environ.get('TSB_FORCE_DISTRIBUTED') == '1'
        if not self.distributed:
            self.devices = parse_devices(self.args.devices)
            return
        self.world_size = int(world)
        self.local_rank = int(os.environ.get('LOCAL_RANK', self.args.local_rank))
        on_gpu = torch.cuda.is_available()
        if on_gpu:
            torch.cuda.set_device(self.local_rank)
        if not dist.is_initialized():
            dist.init_process_group(backend="nccl" if on_gpu else "gloo", init_method='env://')
        self.devices = list(range(self.world_size))

    def inject_default_parser(self):
        """the three options every reference train.py expects (engine.py:70-78)"""
        add = self.parser.add_argument
        add('-d', '--devices', default='', help='set data parallel training')
        add('-c', '--continue', type=extant_file, metavar="FILE", dest="continue_fpath",
            help='continue from one certain checkpoint')
        add('--local_rank', default=0, type=int, help='process rank on node')

    def register_state(self, **kwargs):
        self.state.register(**kwargs)

    def update_iteration(self, epoch, iteration):
        self.state.epoch, self.state.iteration = epoch, iteration

    # ------------------------------------------------------------------ checkpoints (engine.py:89-152)
    def save_checkpoint(self, path):
        """writes {'model', 'optimizer', 'epoch', 'iteration'}"""
        logger.info("Saving checkpoint to file {}".format(path))
        tic = time.time()
        snapshot = dict(model=_portable_state_dict(self.state.model), optimizer=self.state.optimizer.state_dict(),
                        epoch=self.state.epoch, iteration=self.state.iteration)
        mid = time.time()
        torch.save(snapshot, path)
        logger.info("Save checkpoint to file {}, Time usage:\n\tprepare snapshot: {}, IO: {}".format(
            path, mid - tic, time.time() - mid))

    def save_and_link_checkpoint(self, snapshot_dir, log_dir, log_dir_link):
        """epoch-N.pth plus the epoch-last.pth link, and the log-directory link on first use"""
        ensure_dir(snapshot_dir)
        if not osp.exists(log_dir_link):
            link_file(log_dir, log_dir_link)
        target = osp.join(snapshot_dir, 'epoch-{}.pth'.format(self.state.epoch))
        self.save_checkpoint(target)
        link_file(target, osp.join(snapshot_dir, 'epoch-last.pth'))

    def restore_checkpoint(self):
        """resume from `-c FILE`: weights (adding / stripping the `module.` prefix as the live model needs), optimiser
        state, epoch + 1, iteration"""
        tic = time.time()
        blob = torch.load(self.continue_state_object, map_location=torch.device('cpu'), weights_only=False)
        mid = time.time()
        wrapped = any(k.startswith('module.') for k in self.state.model.state_dict())
        self.state.model = load_model(self.state.model, blob['model'], wrapped)
        self.state.optimizer.load_state_dict(blob['optimizer'])
        self.state.epoch, self.state.iteration = blob['epoch'] + 1, blob['iteration']
        del blob
        logger.info("Load checkpoint from file {}, Time usage:\n\tIO: {}, restore snapshot: {}".format(
            self.continue_state_object, mid - tic, time.time() - mid))

    def __enter__(self):
        return self

    def __exit__(self, exc_type, exc_value, tb):
        if torch.cuda.is_available():
            torch.cuda.empty_cache()
        if exc_type is not None:
            logger.warning("A exception occurred during Engine initialization, give up running process")
            return False
