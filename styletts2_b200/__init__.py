"""styletts2_b200: H100 (sm_90a) kernels for the StyleTTS 2 text->waveform inference hot path,
behind the reference's module / notebook interfaces.  See DESIGN.md and INTEGRATION.md."""
__version__ = "0.1.0"
