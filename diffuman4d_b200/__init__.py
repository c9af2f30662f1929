"""diffuman4d_b200 -- Hopper-native (sm_90a, H100) denoise-step hot path for Diffuman4D."""
from .config import UNetConfig, SchedulerConfig  # noqa: F401
