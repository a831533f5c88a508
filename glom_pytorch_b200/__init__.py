"""H100-native (sm_90a) GLOM column-update engine behind the glom-pytorch `Glom` API."""
from ._native import GlomB200Error, LIB_PATH
from .glom import Glom
from .islands import IslandTracks, Islands, ParseTree, islands, parse_tree, track_islands
from . import ops  # noqa: F401  (registers the glom_b200 custom ops, so a saved ExportedProgram loads)

__all__ = ["Glom", "GlomB200Error", "LIB_PATH", "Islands", "islands", "ParseTree", "parse_tree", "IslandTracks",
           "track_islands"]
