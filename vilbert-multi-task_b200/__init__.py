"""vilbert_b200: H100-native (sm_90a) ViLBERT multi-task forward behind the reference worker's object protocol.

Import as ``vilbert_b200`` (the directory name ``vilbert-multi-task_b200`` is not a Python identifier; the
top-level ``vilbert_b200.py`` maps the name onto this package).
"""
from .config import BertConfig
from .model import VILBertForVLTasks
from .pretraining import BertForMultiModalPreTraining
from ._lib import (VilbertB200Error, LIB_PATH, OUT_ALL, OUT_TASK_HEADS, OUT_VIL_PREDICTION,
                   OUT_VIL_PREDICTION_GQA, OUT_VIL_LOGIT, OUT_VIL_BINARY_PREDICTION, OUT_VIL_TRI_PREDICTION,
                   OUT_VISION_PREDICTION, OUT_VISION_LOGIT, OUT_LINGUISIC_PREDICTION, OUT_LINGUISIC_LOGIT)

__all__ = ["BertConfig", "VILBertForVLTasks", "BertForMultiModalPreTraining", "VilbertB200Error", "LIB_PATH"]
