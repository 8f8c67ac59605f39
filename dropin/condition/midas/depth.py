"""Drop-in shim: `from condition.midas.depth import MidasDetector` (reference condition/midas/depth.py) resolves to the GPU
implementation without importing timm.  There is deliberately no __init__.py here: `condition.midas` stays a namespace package."""
from controlar_b200.condition.midas import DPTDepthModel, MidasDetector  # noqa: F401
