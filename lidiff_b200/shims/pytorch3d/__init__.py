"""Minimal stand-in for pytorch3d 0.7.1: `pytorch3d.loss.chamfer_distance` (lidiff/models/models_refine.py:11) on the GPU."""
__version__ = "0.7.1+lidiff_b200.shim"
