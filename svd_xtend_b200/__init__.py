"""svd_xtend_b200 — H100-native (sm_90a) implementation of the SVD spatio-temporal UNet hot path
of pixeli99/SVD_Xtend (the forward/backward step train_svd.py loops over)."""

__version__ = "0.1.0"
