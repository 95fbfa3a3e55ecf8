"""Evaluation of a frozen backbone: k-NN classification on the normalised class token (`knn`), over image datasets
read on the host (`datasets`)."""
from .datasets import ImageFolder, NpzDataset, make_eval_dataset
from .knn import KnnClassifier, eval_knn, extract_features

__all__ = ["ImageFolder", "NpzDataset", "make_eval_dataset", "KnnClassifier", "eval_knn", "extract_features"]
