"""GPU: guided matching through openMVG's own types.  oracle/_ref/dropin_guided_test (built from the reference's sources in
place + host/GeometricFilter_B200.hpp) runs the reference's ImageCollectionGeometricFilter::Robust_model_estimation(functor,
putative, true, ratio) and ImageCollectionGeometricFilter_B200::Robust_model_estimation_{F,E,H}(..., true, ratio) for F
(0.6), E (0.6), H (0.6) and H (-1; the expectation composed from the reference's own pieces, whose PointsToMat cannot run)
on one SfM_Data: a radial-K1 view, two different pinhole intrinsics, a view without an
intrinsic, features at duplicated coordinates and a pair that fails the robust estimation."""
import os
import subprocess

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "oracle", "_ref", "dropin_guided_test")


@pytest.mark.skipif(not os.path.exists(EXE), reason="oracle/_ref/dropin_guided_test not built (needs the openMVG sources at build time)")
def test_guided_matching_dropin_through_openmvg_types():
    p = subprocess.run([EXE], capture_output=True, text=True, timeout=900)
    print(p.stdout[-3000:], p.stderr[-2000:])
    assert p.returncode == 0 and "DROPIN OK" in p.stdout
    for name in ("F, ratio 0.6", "E, ratio 0.6", "H, ratio 0.6", "H, ratio -1"):
        line = next(l for l in p.stdout.splitlines() if f"GUIDED MATCHING ({name})" in l)
        assert "IDENTICAL" in line
