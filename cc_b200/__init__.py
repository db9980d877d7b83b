"""cc_b200: H100-native (sm_90a) implementation of the Competitive-Collaboration
training step's dense per-pixel path, behind the reference's own Python signatures."""
__version__ = "0.1.0"
