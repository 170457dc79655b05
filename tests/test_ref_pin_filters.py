"""The FP64 oracle of the bilateral filter and of the unfiltered mode (oracle/filter_oracle.py) against the compiled reference's own
CostVolumeEnergy ("BL" / "") and NaiveStereoEnergy ("BF" / ""), BilateralFilter included (oracle/_ref/liblexp_ref_filters.so, built
from the reference's headers over oracle/cvshim): filterRects at every corner, inside the image and over all of it, 1x1 and larger
targets, steep / NaN / inf planes, both views, with and without the check, windR 2 / 5 / 20 / 21, MIN_DISPARITY != 0, the cones crop.
Cost-volume "" bit for bit, image-based "" within 1e-4 relative, bilateral within 1e-5 sum w |p|."""
import pytest

from oracle import ref_filters
import filter_checks as FC

pytestmark = pytest.mark.skipif(not ref_filters.available(), reason="oracle/_ref/liblexp_ref_filters.so is not built (needs the reference sources)")
KINDS = [("cv", "bl"), ("cv", "none"), ("naive", "bl"), ("naive", "none")]


@pytest.mark.parametrize("energy,filt", KINDS)
@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("windR", [2, 5, 20, 21])
def test_oracle_equals_reference(energy, filt, mode, windR):
    FC.check_against_reference(energy, filt, 47, 61, 10, windR, mode=mode, seed=windR + mode)


@pytest.mark.parametrize("filt", ["bl", "none"])
def test_oracle_equals_reference_min_disparity(filt):
    FC.check_against_reference("cv", filt, 30, 44, 14, 5, MIN=2.0, MAX=9.5, seed=3)


@pytest.mark.parametrize("energy,filt", KINDS)
@pytest.mark.parametrize("mode", [0, 1])
def test_oracle_equals_reference_on_cones(energy, filt, mode):
    FC.check_against_reference(energy, filt, 0, 0, 20, 10, mode=mode, scene=FC.cones_scene())
