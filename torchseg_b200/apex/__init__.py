"""Shim for `from apex.parallel import DistributedDataParallel, SyncBatchNorm`
(TorchSeg model/bisenet/cityscapes.bisenet.R18/train.py:24-28). Put `torchseg_b200` on sys.path
ahead of a real apex (or import torchseg_b200.apex.parallel directly)."""
