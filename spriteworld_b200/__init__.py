"""spriteworld_b200: H100-native batched Spriteworld step+render engine."""
__version__ = '0.1.0'
