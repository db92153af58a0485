"""get_logger with the reference's behaviour (TorchSeg furnace/engine/logger.py:82-99): root logger,
level from ENGINE_LOGGING_LEVEL, optional file handler, coloured stream handler."""
import logging
import os

from ..utils import pyt_utils

_level = logging.getLevelName(os.getenv('ENGINE_LOGGING_LEVEL', 'INFO').upper())
_COLORS = {logging.DEBUG: ('\x1b[36m', 'DBG '), logging.WARNING: ('\x1b[1;31m', 'WRN '),
           logging.ERROR: ('\x1b[1;4;31m', 'ERR ')}


class LogFormatter(logging.Formatter):
    log_fout = None

    def format(self, record):
        color, tag = _COLORS.get(record.levelno, ('', ''))
        stamp = self.formatTime(record, self.datefmt)
        msg = record.getMessage()
        if self.log_fout:
            return '[%s %d@%s:%s] %s%s' % (stamp, record.lineno, record.filename, record.name, tag, msg)
        end = '\x1b[0m' if color else ''
        return '\x1b[32m%s\x1b[0m %s%s%s%s' % (stamp, color, tag, msg, end)


def get_logger(log_dir=None, log_file=None, formatter=LogFormatter):
    logger = logging.getLogger()
    logger.setLevel(_level)
    del logger.handlers[:]
    if log_dir and log_file:
        pyt_utils.ensure_dir(log_dir)
        LogFormatter.log_fout = True
        fh = logging.FileHandler(log_file, mode='a')
        fh.setLevel(logging.INFO)
        fh.setFormatter(formatter())
        logger.addHandler(fh)
    sh = logging.StreamHandler()
    sh.setFormatter(formatter(datefmt='%d %H:%M:%S'))
    sh.setLevel(0)
    logger.addHandler(sh)
    return logger
