"""Cross-check of the oracle against what the REAL reference computed on seeded random
inputs beyond the cascade goldens (tests/golden/reference_live.npz, recorded by
oracle/make_golden_live.py).  CPU only, bit-exact like tests/test_oracle_golden.py."""
import pytest
import torch

from oracle import casmvs_oracle as O
from oracle.live_inputs import feature_input, predict_depth_inputs


@pytest.mark.parametrize("G", [1, 4])
def test_predict_depth_matches_reference(golden, G):
    from oracle.make_golden import seeded_state_dict
    g = golden("reference_live")
    sd = seeded_state_dict((8, 32, 48), (1, 2, 4), G, seed=5)
    feats, pms, dv = predict_depth_inputs()
    with torch.no_grad():
        d_o, c_o = O.predict_depth(feats, pms, dv, sd, "cost_reg_1.", G)
    assert torch.equal(g[f"depth_g{G}"], d_o) and torch.equal(g[f"confidence_g{G}"], c_o)


def test_feature_pyramid_matches_reference(golden):
    from oracle.make_golden import seeded_state_dict
    g = golden("reference_live")
    sd = seeded_state_dict((8, 32, 48), (1, 2, 4), 1, seed=2)
    with torch.no_grad():
        b = O.feature_pyramid(feature_input(), sd)
    keys = [k[len("feature."):] for k in g if k.startswith("feature.")]
    assert sorted(keys) == sorted(b)
    for k in keys:
        assert torch.equal(g["feature." + k], b[k])
