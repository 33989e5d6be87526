"""GPU: the essential-matrix filter through openMVG's own types.  oracle/_ref/dropin_essential_test (built from the
reference's sources in place + host/GeometricFilter_B200.hpp) runs the reference's
ImageCollectionGeometricFilter::Robust_model_estimation(GeometricFilter_EMatrix_AC(4.0, 2048)) and
ImageCollectionGeometricFilter_B200::Robust_model_estimation_E on one SfM_Data: a radial-K1 view, two different pinhole
intrinsics, a view without an intrinsic, a spherical view and a pair with too few matches."""
import os
import subprocess

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "oracle", "_ref", "dropin_essential_test")


@pytest.mark.skipif(not os.path.exists(EXE), reason="oracle/_ref/dropin_essential_test not built (needs the openMVG sources at build time)")
def test_essential_filter_dropin_through_openmvg_types():
    p = subprocess.run([EXE], capture_output=True, text=True, timeout=600)
    print(p.stdout[-2000:], p.stderr[-2000:])
    assert p.returncode == 0 and "DROPIN OK" in p.stdout
    assert "GEOMETRIC FILTER (E, AC-RANSAC) drop-in" in p.stdout and "IDENTICAL" in p.stdout
