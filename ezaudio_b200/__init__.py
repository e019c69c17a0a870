"""ezaudio_b200 -- H100-native (sm_90a) implementation of EzAudio's DiT-denoise + VAE-decode hot path.

Python host code mirrors the reference's call surface (api/ezaudio.py, api/controlnet.py,
src/models/conditioners.py::MaskDiT, src/modules/autoencoder_wrapper.py::Autoencoder) and calls
hand-written CUDA through the C-ABI library `libezb200.so` (include/ezb200.h).  There is no CPU
or PyTorch fallback: importing the compute modules without the built library raises.
"""
__version__ = "0.1.0"
