"""furniture_b200: H100-native (sm_90a) batched physics backend for the furniture-assembly env hot path."""
__version__ = "0.1.0"
