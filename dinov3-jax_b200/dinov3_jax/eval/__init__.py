"""Evaluation of a frozen backbone: k-NN classification on the normalised class token (`knn`), the linear probe on
class tokens and the patch mean (`linear`), the linear segmentation probe on the patch tokens (`segmentation`), the
linear depth probe on the patch and class tokens (`depth`), video object segmentation by label propagation through the
patch tokens (`video`), keypoint correspondence by nearest neighbour over the upsampled patch tokens
(`correspondence`), unsupervised object discovery by TokenCut's normalized cut on the patch tokens (`discovery`),
instance retrieval by the multi-scale class token on revisited Oxford / Paris (`retrieval`), multinomial logistic
regression on the class token over a grid of regularisation strengths (`logreg`), video classification by an attentive
probe over the frames' patch tokens (`attentive`), over image, video, keypoint-pair, object-box and retrieval datasets
read on the host (`datasets`)."""
from .attentive import AttentiveProbe, eval_attentive
from .correspondence import eval_correspondence
from .datasets import (ADE20KSegmentation, CorrespondenceNpzDataset, DavisDataset, DepthListDataset, DepthNpzDataset,
                       DiscoveryNpzDataset, ImageFolder, NpzDataset, RetrievalNpzDataset, RevisitedDataset,
                       SegNpzDataset, SPairDataset, VideoClassListDataset, VideoClassNpzDataset, VideoNpzDataset,
                       VOCDiscoveryDataset, make_correspondence_dataset, make_depth_dataset, make_discovery_dataset,
                       make_eval_dataset, make_retrieval_dataset, make_seg_dataset, make_video_class_dataset,
                       make_video_dataset)
from .discovery import eval_object_discovery
from .depth import DepthLinearHead, depth_metrics, eval_depth, sample_depth_boxes
from .knn import KnnClassifier, eval_knn, extract_features
from .linear import LinearClassifiers, eval_linear
from .logreg import LogRegSweep, eval_log_regression
from .retrieval import eval_instance_retrieval
from .segmentation import SegLinearHead, eval_segmentation
from .video import eval_video_segmentation

__all__ = ["ImageFolder", "NpzDataset", "make_eval_dataset", "KnnClassifier", "eval_knn", "extract_features",
           "LinearClassifiers", "eval_linear", "ADE20KSegmentation", "SegNpzDataset", "make_seg_dataset",
           "SegLinearHead", "eval_segmentation", "DepthNpzDataset", "DepthListDataset", "make_depth_dataset",
           "DepthLinearHead", "sample_depth_boxes", "depth_metrics", "eval_depth", "DavisDataset", "VideoNpzDataset",
           "make_video_dataset", "eval_video_segmentation", "SPairDataset", "CorrespondenceNpzDataset",
           "make_correspondence_dataset", "eval_correspondence", "VOCDiscoveryDataset", "DiscoveryNpzDataset",
           "make_discovery_dataset", "eval_object_discovery", "RevisitedDataset", "RetrievalNpzDataset",
           "make_retrieval_dataset", "eval_instance_retrieval", "LogRegSweep", "eval_log_regression",
           "VideoClassListDataset", "VideoClassNpzDataset", "make_video_class_dataset", "AttentiveProbe",
           "eval_attentive"]
