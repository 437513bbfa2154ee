"""Log with the contract of util/logger.py:6-17: one INFO file logger per module name writing
./log/<filename>.log relative to the working directory."""
import logging
import os

_FORMAT = "%(asctime)s - %(name)s - %(levelname)s - %(message)s"


def _file_handler(filename):
    os.makedirs("./log/", exist_ok=True)
    h = logging.FileHandler(os.path.join("./log/", filename + ".log"))
    h.setFormatter(logging.Formatter(_FORMAT))
    return h


class Log(object):
    def __init__(self, module, filename, to_file=True):
        self.logger = logging.getLogger(module)
        self.logger.setLevel(logging.INFO)
        if to_file:  # False on the ranks other than 0 of a multi-process run: one log file per run
            self.logger.addHandler(_file_handler(filename))

    def add(self, text):
        self.logger.info(text)
