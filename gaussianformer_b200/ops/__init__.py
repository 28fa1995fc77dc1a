"""Mirror of ``model/encoder/gaussian_encoder/ops/__init__.py:1`` in the reference, plus the opt-in fused
caller path (``deformable_aggregation_fused``, SURVEY.md 8f-2), its variant that projects 3-D key points itself
(``deformable_aggregation_from_key_points``) and the key-point generator in front of it
(``anchor_key_points`` / ``SparseGaussian3DKeyPointsGenerator``), and the encoder's submanifold sparse convolution
(``SparseConv3D`` / ``SubMConv3d`` / ``subm_conv3d``) in place of spconv, and both refinement modules' arithmetic
after their MLP (``gaussian_refine`` / ``SparseGaussian3DRefinementModule`` / ``SparseGaussian3DRefinementModuleV2``)."""
from .deformable_aggregation import (DeformableAggregationFunction, DeformableAggregationFusedFunction,  # noqa: F401
                                     deformable_aggregation_from_key_points, deformable_aggregation_fused, feature_maps_format, fused_supported)
from .key_points import SparseGaussian3DKeyPointsGenerator, anchor_key_points  # noqa: F401
from .refine import (GaussianPrediction, SparseGaussian3DRefinementModule,  # noqa: F401
                     SparseGaussian3DRefinementModuleV2, gaussian_refine)
from .sparse_conv import SparseConv3D, SubMConv3d, SubMConv3dFunction, build_rulebook, subm_conv3d  # noqa: F401

__all__ = ["DeformableAggregationFunction", "feature_maps_format", "DeformableAggregationFusedFunction",
           "deformable_aggregation_fused", "fused_supported", "deformable_aggregation_from_key_points",
           "anchor_key_points", "SparseGaussian3DKeyPointsGenerator", "SparseConv3D", "SubMConv3d", "SubMConv3dFunction",
           "build_rulebook", "subm_conv3d", "gaussian_refine", "GaussianPrediction", "SparseGaussian3DRefinementModule",
           "SparseGaussian3DRefinementModuleV2"]
