"""Former home of depth peeling's CPU ray query -- TEST INFRASTRUCTURE.

The query (closest hit with t > sep(t_prev), ties to the lowest id) now lives in ``oracle/mcoracle.c`` next to ``orc_closest_hit`` and
``orc_rasterize``, wrapped by ``oracle.Scene`` (``closest_hit(ro, rd, t_after)``, ``peel``, ``all_hits``); this module keeps
``PeelScene`` and ``sep`` importable for code written against the earlier layout.  It has no build or library of its own.
"""
from common import oracle
from oracle import peel_sep as sep  # noqa: F401


def PeelScene(verts, tris):
    """The brute-force fp32 oracle scene of (verts, tris)."""
    return oracle().scene(verts, tris)
