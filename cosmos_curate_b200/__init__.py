"""cosmos_curate_b200 - H100-native decode -> sample -> preprocess -> embed/classify path.

Host side mirrors the reference's plugin surface (CuratorStage / ModelInterface); all device work is
hand-written sm_90a CUDA in libcurate_b200.so, bound with ctypes (cosmos_curate_b200/_lib.py).
"""

__version__ = "0.1.0"
