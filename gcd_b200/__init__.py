"""gcd_b200 — H100-native (sm_90a) denoising hot path for Generative Camera Dolly (basilevh/gcd)."""
__version__ = "0.1.0"
