"""Shim for dense_correspondence/evaluation/evaluation.py -> this project's implementation (per-match statistics only)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import _load  # noqa: F401
from pdc_b200.evaluation import (DenseCorrespondenceEvaluation, DCNEvaluationPandaTemplate, PandaDataFrameWrapper,  # noqa: F401
                                 match_statistics, quantitative_analysis_on_pair)
