"""controlar_b200 — H100-native (sm_90a) implementation of ControlAR's conditional-decoding hot path behind the
reference's own Python API.  See DESIGN.md / INTEGRATION.md."""
__version__ = "0.1.0"
