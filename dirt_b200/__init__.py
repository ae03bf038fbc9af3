"""dirt_b200 -- an H100-native (sm_90a) differentiable rasteriser behind the dirt.rasterise API.

`import dirt_b200 as dirt` is the drop-in for the reference package (dirt/__init__.py:1-3).
"""
from .rasterise_ops import rasterise, rasterise_batch, rasterise_deferred, rasterise_batch_deferred
from .texture import (index_derivatives, latlong_directions, latlong_to_cubemap, sample_cubemap, sample_texture,
                      uvs_to_pixel_indices)
from . import matrices, lighting, mesh, projection

__all__ = ['rasterise', 'rasterise_batch', 'rasterise_deferred', 'rasterise_batch_deferred',
           'sample_texture', 'sample_cubemap', 'latlong_to_cubemap', 'latlong_directions', 'uvs_to_pixel_indices',
           'index_derivatives', 'matrices', 'lighting', 'mesh', 'projection']
