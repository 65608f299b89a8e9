"""jukebox_b200 - H100-native (sm_90a) implementation of Jukebox's sampling hot path:
autoregressive prior decode + VQ-VAE encode/decode, behind the reference's
hparams / make_models / sample surface.  All arithmetic is in libjkb200.so
(jukebox_b200/csrc, C ABI in include/jkb200.h); there is no CPU or eager-PyTorch path."""
__version__ = "0.1.0"
