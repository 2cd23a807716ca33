"""wide_deep_b200 — H100-native (sm_90a) Wide&Deep CTR train/eval hot path (drop-in for Lapis-Hong/wide_deep's
conf/*.yaml surface and python/train.py | eval.py entry points).  See DESIGN.md."""
__version__ = "0.1.0"
