"""H100-native (sm_90a) GLOM column-update engine behind the glom-pytorch `Glom` API."""
from ._native import GlomB200Error, LIB_PATH
from .glom import Glom
from .islands import Islands, islands

__all__ = ["Glom", "GlomB200Error", "LIB_PATH", "Islands", "islands"]
