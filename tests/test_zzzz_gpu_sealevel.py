"""GPU: a varying sea surface height (tests/sealevelcases.py: runs of the unmodified reference) through the drop-in OceanDrift --
the water column in the sea-floor interaction, buoyancy and mixing, drift:vertical_advection_correction and its previous-step
store, on the device."""
import pytest

import sealevelcases as sc

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('case', list(sc.CASES))
def test_sea_level_case_equals_the_reference(case):
    o = sc.run_product(case)
    n_act, n_deact, cats = sc.check(o, case)
    print(case, n_act, n_deact, cats)
