from .heatmap import HeatmapHead  # noqa: F401
from .heatmap_mhcrnn import HeatmapMHCRNNHead, UpsamplingCRNN  # noqa: F401
from .regression import LinearRegressionHead  # noqa: F401
