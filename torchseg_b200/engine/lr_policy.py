"""Learning-rate schedules with the reference's class names and `get_lr(step)` protocol
(TorchSeg furnace/engine/lr_policy.py:11-49). Each schedule is a small callable table: the train loops only
ever call `policy.get_lr(iteration)` (train.py:133) and read nothing else, except `PolyLR.start_lr / lr_power /
total_iters`, which stay public."""


class BaseLR(object):
    """protocol: get_lr(position) → float"""

    def get_lr(self, position):
        raise NotImplementedError("%s does not define get_lr" % type(self).__name__)

    __call__ = lambda self, position: self.get_lr(position)


class PolyLR(BaseLR):
    """polynomial decay to zero: start_lr · (1 − it / total_iters) ** lr_power   (lr_policy.py:18-26)"""

    def __init__(self, start_lr, lr_power, total_iters):
        self.start_lr, self.lr_power, self.total_iters = start_lr, lr_power, float(total_iters)

    def get_lr(self, cur_iter):
        remaining = 1.0 - float(cur_iter) / self.total_iters
        return self.start_lr * remaining ** self.lr_power


class MultiStageLR(BaseLR):
    """piecewise-constant schedule from `[(until_iter, lr), ...]`: the lr of the first stage whose bound lies beyond
    the position; None past the last bound, like the reference (lr_policy.py:29-38)"""

    def __init__(self, lr_stages):
        ok = isinstance(lr_stages, (list, tuple)) and len(lr_stages) > 0 and len(lr_stages[0]) == 2
        if not ok:
            raise AssertionError('lr_stages must be list or tuple, with [iters, lr] format')
        self._stages = [(bound, lr) for bound, lr in lr_stages]

    def get_lr(self, epoch):
        return next((lr for bound, lr in self._stages if epoch < bound), None)


class LinearIncreaseLR(BaseLR):
    """linear warm-up from start_lr towards end_lr over warm_iters positions (lr_policy.py:41-49)"""

    def __init__(self, start_lr, end_lr, warm_iters):
        self._origin = start_lr
        self._slope = (end_lr - start_lr) / warm_iters

    def get_lr(self, cur_epoch):
        return self._origin + self._slope * cur_epoch
