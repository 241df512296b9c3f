"""denseflow_b200 — H100-native (sm_90a) dense optical flow behind the call boundary of open-mmlab/denseflow's
hot path (cv::cuda::OpticalFlowDual_TVL1 / FarnebackOpticalFlow ::calc at src/denseflow_gpu.cpp:327,329)."""
from .api import DenseOpticalFlow, FarnebackOpticalFlow, OpticalFlowDual_TVL1, create  # noqa: F401

__all__ = ["DenseOpticalFlow", "OpticalFlowDual_TVL1", "FarnebackOpticalFlow", "create"]
