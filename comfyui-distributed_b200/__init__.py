"""comfyui-distributed_b200 -- H100-native drop-in for the Ultimate-SD-Upscale tile hot
path of ComfyUI-Distributed (tile scatter -> per-tile denoise -> gather -> seam blend).

ComfyUI loads this directory as a custom node package and reads NODE_CLASS_MAPPINGS
(reference: __init__.py:17-26, nodes/__init__.py:14-15, nodes/distributed_upscale.py:273-279).
"""
from .nodes import NODE_CLASS_MAPPINGS, NODE_DISPLAY_NAME_MAPPINGS
from .http_master import install_in_comfyui as _install_routes

_install_routes()      # inside ComfyUI: serve the masters' routes (http_master.py, http_collector.py, orchestrator.py)

__all__ = ["NODE_CLASS_MAPPINGS", "NODE_DISPLAY_NAME_MAPPINGS"]
