"""slamkit_b200 -- H100-native (sm_90a) hot paths of slp-rl/slamkit behind the reference's plugin interfaces.

Only what the two hot paths need lives here:
  csrc/                hand-written CUDA kernels + the C ABI (libslamkit_b200.so, include/slamkit_b200.h)
  _lib.py, ops.py      ctypes binding; one wrapper per op-level entry point
  lm.py                B200UnitLM / B200AdamW: mirror of slamkit.model (TokenLM plugin, tlm_type="b200")
  feature_extractor.py HubertB200FeatureExtractor: mirror of slamkit.feature_extractor (feature_extractor_type="hubert_b200")
  tokeniser.py         UnitTokeniser mirror (dedup, <Un{i}> strings, ids)
"""
__version__ = "0.1.0"
