"""H100-native differentiable primitive renderer: drop-in for the render hot path of
monniert/differentiable-blocksworld (see DESIGN.md).  Import as `dbw_b200` (alias module at the repo root)."""
from . import _lib                                   # noqa: F401
from .structures import Meshes, TexturesUV, join_meshes_as_scene, join_meshes_as_batch   # noqa: F401
from .renderer import Renderer, render_scene                                              # noqa: F401

__all__ = ['Meshes', 'TexturesUV', 'join_meshes_as_scene', 'join_meshes_as_batch', 'Renderer', 'render_scene']
