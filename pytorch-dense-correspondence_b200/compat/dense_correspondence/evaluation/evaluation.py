"""Shim for dense_correspondence/evaluation/evaluation.py -> this project's implementation (per-match statistics, descriptor statistics, across-object analysis)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import _load  # noqa: F401
from pdc_b200.evaluation import (DenseCorrespondenceEvaluation, DCNEvaluationPandaTemplate, PandaDataFrameWrapper,  # noqa: F401
                                 DCNEvaluationPandaTemplateAcrossObject, match_statistics, quantitative_analysis_on_pair,
                                 descriptor_statistics, descriptor_statistics_over_images, save_descriptor_statistics,
                                 across_object_analysis)
