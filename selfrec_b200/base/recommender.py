"""Lifecycle base class with the attribute surface of base/recommender.py:7-83.

Only what GraphRecommender and the in-scope models rely on: config unpacking (table-driven here), the
build -> train -> test -> evaluate template, and the log handle."""
import os
import time

from ..data.data import Data
from ..shard_rank import is_main_process
from ..util.logger import Log

# attribute, YAML key, conversion, label printed by print_model_info (None: not printed)
_SETTINGS = (
    ("ranking", "item.ranking.topN", lambda v: v, None),
    ("emb_size", "embedding.size", int, "Embedding Dimension:"),
    ("maxEpoch", "max.epoch", int, "Maximum Epoch:"),
    ("lRate", "learning.rate", float, "Learning Rate:"),
    ("batch_size", "batch.size", int, "Batch Size:"),
    ("reg", "reg.lambda", float, "Regularization Parameter:"),
    ("output", "output", lambda v: v, None),
)
_STAGES = (("Initializing and building model...", "build"), ("Training Model...", "train"))


def _noop(self, *args, **kwargs):
    return None


class Recommender:
    def __init__(self, conf, training_set, test_set, **kwargs):
        self.config = conf
        self.data = Data(conf, training_set, test_set)
        self.model_name = conf["model"]["name"]
        for attr, key, cast, _label in _SETTINGS:
            setattr(self, attr, cast(conf[key]))
        now = time.strftime("%Y-%m-%d %H-%M-%S", time.localtime(time.time()))
        self.model_log = Log(self.model_name, self.model_name + " " + now, to_file=is_main_process())
        self.result, self.recOutput = [], []

    def initializing_log(self):
        log = self.model_log.add
        log("### model configuration ###")
        for key, value in self.config.config.items():
            log(f"{key}={value}")

    def print_model_info(self):
        conf = self.config
        rows = [("Model:", self.model_name)]
        rows += [(label, os.path.abspath(conf[key])) for label, key in (("Training Set:", "training.set"), ("Test Set:", "test.set"))]
        rows += [(label, getattr(self, attr)) for attr, _key, _cast, label in _SETTINGS if label]
        for label, value in rows:
            print(label, value)
        if conf.contain(self.model_name):
            extra = conf[self.model_name]
            print("Specific parameters:", "  ".join(f"{k}:{extra[k]}" for k in extra))

    # hooks the concrete models fill in
    build = train = predict = test = save = load = evaluate = _noop

    def execute(self):
        self.initializing_log()
        self.print_model_info()
        for banner, stage in _STAGES:
            print(banner)
            getattr(self, stage)()
        print("Testing...")
        rec_list = self.test()
        print("Evaluating...")
        self.evaluate(rec_list)
