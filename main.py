"""python main.py [--key=value ...] -- the reference's driver (main.py:1-45) without TensorFlow.

Reads NeuRec.properties (+ conf/<recommender>.properties), builds the Dataset, resolves the
model class by name and runs build_graph() / train_model() on the sm_90a kernels.
"""
import importlib
import os
import random
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from neurec_b200.data.dataset import Dataset  # noqa: E402
from neurec_b200.util import Configurator  # noqa: E402

np.random.seed(2018)      # main.py:10
random.seed(2018)         # main.py:11  (tf.set_random_seed(2017) -> model init generators use 2017)


def resolve_model(recommender):
    # main.py:30-40: general_recommender first, then social_recommender, then sequential_recommender; only the models
    # listed below are on the accelerated hot path
    for family in ("general_recommender", "social_recommender", "sequential_recommender"):
        name = "neurec_b200.model.%s.%s" % (family, recommender)
        if importlib.util.find_spec(name) is not None:
            return getattr(importlib.import_module(name), recommender)
    raise ImportError("recommender '%s' is outside the accelerated hot path "
                      "(available: MF, MLP, NeuMF, LightGCN, NGCF, APR, SpectralCF, WRMF, SBPR, FPMC, TransRec, "
                      "HRM, NPE, FPMCplus, Caser, FISM, ItemKNN)" % recommender)


if __name__ == "__main__":
    conf = Configurator("NeuRec.properties", default_section="hyperparameters")
    os.environ["CUDA_VISIBLE_DEVICES"] = str(conf["gpu_id"])      # main.py:17-18
    import torch
    torch.cuda.init()
    dataset = Dataset(conf)
    Model = resolve_model(conf["recommender"])
    model = Model(None, dataset, conf)                            # sess=None: no TF session
    model.build_graph()
    model.train_model()
