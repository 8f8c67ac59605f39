"""Drop-in shim: `from condition.lineart import LineArt` (reference condition/lineart.py) resolves to the GPU implementation, without
the reference's unused `controlnet_aux` import."""
from controlar_b200.condition.lineart import *  # noqa: F401,F403
from controlar_b200.condition.lineart import LineArt, ResidualBlock  # noqa: F401
