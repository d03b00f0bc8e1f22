"""Import-path shim: `microwakeword.inference` / `microwakeword.audio.audio_utils` resolve to the
H100 implementation so reference call sites (test.py:321-336, :434) run unchanged."""
