"""GPU: the angular essential-matrix filters (`-g a`, `-g u`) through openMVG's own types.  oracle/_ref/dropin_angular_test
(built from the reference's sources in place + host/GeometricFilter_B200.hpp) runs the reference's
ImageCollectionGeometricFilter::Robust_model_estimation(GeometricFilter_ESphericalMatrix_AC_Angular<false | true>(4.0, 2048))
and ImageCollectionGeometricFilter_B200::Robust_model_estimation_EAngular / _EUpright on one SfM_Data, with guided
matching off and on: spherical views, a radial-K1 view, two different pinhole intrinsics, a view without an intrinsic
and a pair at the keep threshold for each model."""
import os
import subprocess

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "oracle", "_ref", "dropin_angular_test")


@pytest.mark.skipif(not os.path.exists(EXE), reason="oracle/_ref/dropin_angular_test not built (needs the openMVG sources at build time)")
def test_angular_filters_dropin_through_openmvg_types():
    p = subprocess.run([EXE], capture_output=True, text=True, timeout=600)
    print(p.stdout[-3000:], p.stderr[-2000:])
    assert p.returncode == 0 and "DROPIN OK" in p.stdout
    lines = [l for l in p.stdout.splitlines() if "drop-in:" in l]
    assert len(lines) == 4 and all("IDENTICAL" in l and "NOT KEPT" not in l for l in lines)
