"""macaw-llm_b200 — H100-native (sm_90a) implementation of the Macaw-LLM `MM_LLMs` forward hot path.

Layout
  csrc/      hand-written CUDA kernels + the C ABI (include/macaw_b200.h)  -> libmacaw_b200.so
  _lib.py    ctypes loader / signature table
  ops.py     torch-tensor front end of the C ABI
  engine.py  the forward pass expressed over those ops (encoders, alignment, splice, LLaMA)
  modeling.py  drop-in `MM_LLMs` / `MM_LLMs_Config` class surface (reference: modeling.py:807-1093)
"""
__version__ = "0.1.0"
