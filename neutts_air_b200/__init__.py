"""neutts_air_b200 — H100 (sm_90a) implementation of NeuTTS-Air's two inference hot paths
(speech-LM prefill/decode and the NeuCodec decoder) behind a C-ABI shared library.

Only what the path needs lives here: ``csrc/`` (CUDA kernels + C-ABI), ``_lib`` (ctypes binding),
``lm`` / ``codec`` (host-side engines mirroring the reference's two inner seams), ``loader``
(checkpoint readers), ``dist`` (utterance sharding + the one NCCL all-gather).  The drop-in
``neutts.NeuTTS`` facade lives in the top-level ``neutts`` package.
"""
__version__ = "0.1.0"
