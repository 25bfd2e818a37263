"""AbstractRecommender: the model plug-in base classes (reference model/AbstractRecommender.py:9-80): the general
base, the sequential base (models that need the interaction times) and the social base."""
import os
import time

import numpy as np
import pandas as pd
import scipy.sparse as sp

from ..evaluator import ProxyEvaluator
from ..util.logger import Logger

# ProxyEvaluator keyword <- configuration key (AbstractRecommender.py:25-32)
_EVALUATOR_OPTIONS = (("metric", "metric"), ("group_view", "group_view"), ("top_k", "topk"),
                      ("batch_size", "test_batch_size"), ("num_thread", "num_thread"))


def _create_logger(config, data_name):
    # AbstractRecommender.py:9-20: log/<dataset>/<model>/<dataset>_<params[:150]>_<ts>.log
    run_id = "%s_%.8f" % (("%s_%s" % (data_name, config.params_str()))[:150], time.time())
    return Logger(os.path.join("log", data_name, config["recommender"], run_id + ".log"))


class AbstractRecommender(object):
    """Every model gets its evaluator (train / test / negative-test dicts of the dataset + the
    evaluation options of NeuRec.properties) and its logger, and logs dataset and configuration."""

    def __init__(self, dataset, conf):
        splits = (dataset.get_user_train_dict(), dataset.get_user_test_dict(), dataset.get_user_test_neg_dict())
        options = {kw: conf[key] for kw, key in _EVALUATOR_OPTIONS}
        self.evaluator = ProxyEvaluator(*splits, **options)
        self.logger = _create_logger(conf, dataset.dataset_name)
        for what in (dataset, conf):
            self.logger.info(what)

    def build_graph(self):
        raise NotImplementedError

    def train_model(self):
        raise NotImplementedError

    def predict(self, user_ids, items):
        raise NotImplementedError


class SeqAbstractRecommender(AbstractRecommender):
    """AbstractRecommender.py:48-52: a sequential model needs the dataset's time matrix (a UIRT or UIT column
    format); without it the constructor fails before the evaluator and the logger are built."""

    def __init__(self, dataset, conf):
        if dataset.time_matrix is None:
            raise ValueError("Dataset does not contant time infomation!")
        super(SeqAbstractRecommender, self).__init__(dataset, conf)


class SocialAbstractRecommender(AbstractRecommender):
    """AbstractRecommender.py:54-74: reads conf["social_file"] (user, friend pairs in raw ids), keeps the pairs whose
    two ends are known users and builds ``social_matrix`` (users x users CSR; duplicate pairs collapse)."""

    def __init__(self, dataset, conf):
        super(SocialAbstractRecommender, self).__init__(dataset, conf)
        pairs = pd.read_csv(conf["social_file"], sep=conf["data.convert.separator"], header=None,
                            names=["user", "friend"])
        known = np.array(list(dataset.userids.keys()))
        pairs = pairs[np.isin(pairs["user"], known)]
        pairs = pairs[np.isin(pairs["friend"], known)]
        user_id = [dataset.userids[u] for u in pairs["user"]]
        friend_id = [dataset.userids[u] for u in pairs["friend"]]
        num_users = dataset.train_matrix.shape[0]
        self.social_matrix = sp.csr_matrix(([1] * len(user_id), (user_id, friend_id)), shape=(num_users, num_users))
