"""Evaluation of a frozen backbone: k-NN classification on the normalised class token (`knn`), the linear probe on
class tokens and the patch mean (`linear`), over image datasets read on the host (`datasets`)."""
from .datasets import ImageFolder, NpzDataset, make_eval_dataset
from .knn import KnnClassifier, eval_knn, extract_features
from .linear import LinearClassifiers, eval_linear

__all__ = ["ImageFolder", "NpzDataset", "make_eval_dataset", "KnnClassifier", "eval_knn", "extract_features",
           "LinearClassifiers", "eval_linear"]
