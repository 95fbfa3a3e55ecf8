"""Evaluation of a frozen backbone: k-NN classification on the normalised class token (`knn`), the linear probe on
class tokens and the patch mean (`linear`), the linear segmentation probe on the patch tokens (`segmentation`), over
image datasets read on the host (`datasets`)."""
from .datasets import (ADE20KSegmentation, ImageFolder, NpzDataset, SegNpzDataset, make_eval_dataset,
                       make_seg_dataset)
from .knn import KnnClassifier, eval_knn, extract_features
from .linear import LinearClassifiers, eval_linear
from .segmentation import SegLinearHead, eval_segmentation

__all__ = ["ImageFolder", "NpzDataset", "make_eval_dataset", "KnnClassifier", "eval_knn", "extract_features",
           "LinearClassifiers", "eval_linear", "ADE20KSegmentation", "SegNpzDataset", "make_seg_dataset",
           "SegLinearHead", "eval_segmentation"]
