"""PlenOctree side of the path: svox-compatible N3Tree / VolumeRenderer over the CUDA library, and mirrors of
octree/extraction.py and octree/optimization.py (SURVEY.md §8 rows a13, a15; §8f ranks 2-3)."""
from .n3tree import DataFormat, N3Tree, N3TreeView, QuantTree, load_tree  # noqa: F401
from .renderer import NDCConfig, Rays, VolumeRenderer, disparity  # noqa: F401
