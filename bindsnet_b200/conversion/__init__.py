from .conversion import FeatureExtractor, Permute, ann_to_snn, data_based_normalization
from .nodes import PassThroughNodes, SubtractiveResetIFNodes
from .topology import ConstantPad2dConnection, PermuteConnection

__all__ = [
    "Permute",
    "FeatureExtractor",
    "SubtractiveResetIFNodes",
    "PassThroughNodes",
    "PermuteConnection",
    "ConstantPad2dConnection",
    "data_based_normalization",
    "ann_to_snn",
]
