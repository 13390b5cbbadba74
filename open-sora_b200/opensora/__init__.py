"""Host-side mirror of the reference's `opensora` package for the denoiser / VAE hot path only
(SURVEY.md §8b).  Same module paths, class names, registry keys and state-dict keys as the
reference so its scripts import it unchanged; the arithmetic runs in libosb200.so (sm_90a)."""
