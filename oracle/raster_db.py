"""Former import path of the screen-space-derivative oracle -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

rast_db, interpolate's out_da, their adjoints and interpolate's forward are restated in ``oracle/geometry.c`` and wrapped by
``oracle/geometry.py``; this module keeps ``raster_db_oracle`` importable for code written against the earlier layout.
"""
from oracle.geometry import GeometryOracle as RasterDbOracle, build, geometry_oracle as raster_db_oracle  # noqa: F401
