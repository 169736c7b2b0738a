"""The host tables of the fixed-step backward (``schedule.backward_tables``): the reversed step and stage arrays and the
output gradients every grid state receives, derived here directly from each output's step, mode and slope."""
import pytest
import torch

from test_host_logic import FIXED_SCHEDULES, fixed_schedule_knots
from torchcde_b200 import schedule


def _schedule(sname, method):
    ts, step, uneven = FIXED_SCHEDULES[sname]
    knots = fixed_schedule_knots(uneven)
    t = knots.double() if ts is None else torch.tensor(ts, dtype=torch.float32 if sname == "F4" else torch.float64)
    return schedule.build_schedule(t, knots, knots.numel() - 1, method, step, torch.float32)


@pytest.mark.parametrize("method", ["rk4", "midpoint", "euler"])
@pytest.mark.parametrize("sname", list(FIXED_SCHEDULES))
def test_backward_tables(sname, method):
    s = _schedule(sname, method)
    tab = schedule.backward_tables(s)
    n = s.n_steps
    assert torch.equal(tab["step_dt"], s.step_dt.flip(0))
    assert torch.equal(tab["stage_index"], s.stage_index.reshape(-1).flip(0))
    assert torch.equal(tab["stage_frac"], s.stage_frac.reshape(-1).flip(0))
    rng = tab["inj_range"].tolist()
    assert len(rng) == n + 2 and rng[0] == 0 and rng == sorted(rng) and rng[-1] == tab["inj_out"].numel()
    assert tab["inj_weight"].dtype == torch.float32
    got = {}                                     # output -> {grid state: weight}
    for r in range(n + 1):
        for e in range(rng[r], rng[r + 1]):
            j = int(tab["inj_out"][e])
            state = n - r
            assert state not in got.setdefault(j, {})
            got[j][state] = float(tab["inj_weight"][e])
    assert sorted(got) == list(range(s.n_out))
    for j in range(s.n_out):
        step, mode, slope = int(s.out_step[j]), int(s.out_mode[j]), float(s.out_slope[j])
        if step < 0:
            want = {0: 1.0}
        elif mode == 0:
            want = {step: 1.0}
        elif mode == 1:
            want = {step + 1: 1.0}
        else:
            want = {step: float(torch.tensor(1.0, dtype=torch.float32) - torch.tensor(slope, dtype=torch.float32)),
                    step + 1: slope}
        assert got[j] == want, (j, got[j], want)
        assert abs(sum(got[j].values()) - 1.0) <= 2.0 ** -24
