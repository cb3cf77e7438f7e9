"""Renderers (reference: spriteworld/renderers/__init__.py)."""
from spriteworld_b200.renderers import color_maps  # noqa: F401
from spriteworld_b200.renderers.abstract_renderer import AbstractRenderer  # noqa: F401
from spriteworld_b200.renderers.glimpses import SpriteGlimpses  # noqa: F401
from spriteworld_b200.renderers.glimpses import SpriteLayers  # noqa: F401
from spriteworld_b200.renderers.handcrafted import GoalPositions  # noqa: F401
from spriteworld_b200.renderers.handcrafted import SoftSpriteMasks  # noqa: F401
from spriteworld_b200.renderers.handcrafted import SpriteBoxes  # noqa: F401
from spriteworld_b200.renderers.handcrafted import SpriteCoverage  # noqa: F401
from spriteworld_b200.renderers.handcrafted import SpriteFactors  # noqa: F401
from spriteworld_b200.renderers.handcrafted import SpriteMasks  # noqa: F401
from spriteworld_b200.renderers.handcrafted import SpritePassthrough  # noqa: F401
from spriteworld_b200.renderers.handcrafted import Success  # noqa: F401
from spriteworld_b200.renderers.pil_renderer import PILRenderer  # noqa: F401
