"""CPU: every function an oracle library exports has a declared signature, and every declared signature names an export.  The oracle's
counterpart of test_cabi.py: without a declared signature ctypes checks neither the count nor the types of the arguments."""
import ctypes
import os
import re

import pytest

from oracle import LIBS, REAL, Oracle
from oracle.dmtet import DmtetOracle
from oracle.geometry import GeometryOracle
from oracle.hashgrid import HashGridOracle
from oracle.mipchain import MipChainOracle
from oracle.mlptexture import MlpTextureOracle
from oracle.regularizer import RegularizerOracle
from oracle.taps import TapsOracle
from oracle.texture import TextureOracle

ORACLE_DIR = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle")
WRAPPERS = [(Oracle, 48), (GeometryOracle, 15), (HashGridOracle, 4), (TextureOracle, 4), (MlpTextureOracle, 7),
            (DmtetOracle, 9), (RegularizerOracle, 7), (MipChainOracle, 5), (TapsOracle, 7)]     # exports of each library at the time of writing


def _exports(lib):
    """Names of the non-static orc_* / geo_* / hg_* / tex_* / mlt_* / dmt_* / reg_* / mip_* / taps_* function definitions of every C file
    of a library."""
    names = []
    for source in LIBS[lib]:
        if source.endswith(".c"):
            src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ORACLE_DIR, source)).read(), flags=re.S)
            names += re.findall(r"^(?!static\b)[A-Za-z_][\w \*]*?\b((?:orc|geo|hg|tex|mlt|dmt|reg|mip|taps)_\w+)\s*\([^;{]*\)\s*\{", src, re.M)
    return sorted(names)


def test_every_library_has_a_wrapper():
    assert sorted(cls.LIB for cls, _ in WRAPPERS) == sorted(LIBS)


@pytest.mark.parametrize("cls,n", WRAPPERS, ids=[cls.LIB for cls, _ in WRAPPERS])
def test_signature_table_names_exactly_the_exports(cls, n):
    names = _exports(cls.LIB)
    assert len(names) >= n, "the definition pattern no longer finds the exports"
    assert sorted(cls.SIGS) == names, "signature table and source disagree"


@pytest.mark.parametrize("f64", [False, True])
@pytest.mark.parametrize("cls", [cls for cls, _ in WRAPPERS], ids=[cls.LIB for cls, _ in WRAPPERS])
def test_each_library_loads_once_per_precision_with_its_table(cls, f64):
    o = cls.get(f64)
    assert o is cls.get(f64) and o is not cls.get(not f64) and o.f64 == f64
    for name, (args, res) in cls.SIGS.items():
        fn = getattr(o.lib, name)
        assert fn.restype is res and list(fn.argtypes) == [o.real if a is REAL else a for a in args], name
    assert o.real is (ctypes.c_double if f64 else ctypes.c_float)
