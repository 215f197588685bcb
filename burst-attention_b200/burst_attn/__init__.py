"""burst_attn -- H100-native drop-in for MayDomine/Burst-Attention's import surface
(reference burst_attn/__init__.py:1 re-exports burst_attn_interface)."""
from .burst_attn_interface import *  # noqa: F401,F403
from .burst_attn_interface import burst_attn_func, burst_attn_func_striped  # noqa: F401
