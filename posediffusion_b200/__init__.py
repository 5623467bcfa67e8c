"""posediffusion_b200 -- H100-native (sm_90a) implementation of PoseDiffusion's sampling hot path.

Public surface mirrors the reference's (`models.PoseDiffusionModel`, `models.GaussianDiffusion`,
`models.Denoiser`, `util.geometry_guided_sampling.geometry_guided_sampling`,
`util.camera_transform.pose_encoding_to_camera`); compute goes through the C-ABI library
`libposediff_b200.so` (include/posediff_b200.h).  No CPU or PyTorch-operator fallback exists.
"""
from .camera_alignment import corresponding_cameras_alignment
from .camera_transform import PerspectiveCameras, pose_encoding_to_camera
from .denoiser import Denoiser, TransformerEncoderWrapper
from .gaussian_diffuser import GaussianDiffusion
from .geometry_guided_sampling import geometry_guided_sampling, invalidate_matches
from .image_feature_extractor import MultiScaleImageFeatureExtractor
from .pose_diffusion_model import PoseDiffusionModel

__all__ = [
    "PoseDiffusionModel", "GaussianDiffusion", "Denoiser", "TransformerEncoderWrapper", "MultiScaleImageFeatureExtractor",
    "geometry_guided_sampling", "invalidate_matches", "pose_encoding_to_camera", "PerspectiveCameras", "corresponding_cameras_alignment",
]
