"""The oracle trajectory_ate (tests/ate_oracle.py: scipy.spatial.procrustes restated in torch)
reproduces the reference's compute_ate on tests/golden/ate.npz, including the case where the
reference raises."""
import pytest
import torch

import ate_oracle as O
from ate_checks import check_case, golden_cases

CASES = golden_cases()


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_trajectory_ate_matches_reference(name):
    c = CASES[name]
    gt = torch.as_tensor(c["gt"], dtype=torch.float64)
    pred = torch.as_tensor(c["pred"], dtype=torch.float64)
    ate, al_gt, al_pred, degenerate = O.trajectory_ate(gt, pred)
    assert bool(degenerate) == bool(c["raised"])
    if c["raised"]:
        assert torch.isnan(ate)
        return
    check_case(name, c, ate, al_gt.numpy(), al_pred.numpy())


def test_oracle_trajectory_ate_is_batched():
    names = [n for n in sorted(CASES) if CASES[n]["gt"].shape[0] == 150]
    gt = torch.stack([torch.as_tensor(CASES[n]["gt"], dtype=torch.float64) for n in names])
    pred = torch.stack([torch.as_tensor(CASES[n]["pred"], dtype=torch.float64) for n in names])
    ate, _, _, degenerate = O.trajectory_ate(gt, pred)
    for i, n in enumerate(names):
        one = O.trajectory_ate(gt[i], pred[i])
        assert bool(degenerate[i]) == bool(one[3])
        assert torch.allclose(ate[i], one[0], rtol=1e-9, atol=1e-15, equal_nan=True), n
