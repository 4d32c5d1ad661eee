"""H100-native (sm_90a) DDPM sampling hot path of music-spectrogram-diffusion."""
