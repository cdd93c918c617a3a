"""The conv_tc tile plans are pinned: the library must reproduce tests/golden/conv_tc_plans.json
(the plan line, rc, grid, block and shared memory of every shape and knob set that
tests/golden/make_conv_tc_plans.py records, hashed per group) exactly.  Runs without a GPU, like
test_conv_plan.py.  The grid is min(tiles, SMs) and the table was written for the 132 SMs of an
H100 SXM; on a device with another SM count the grid is left out of the comparison."""
import json

import make_conv_tc_plans as mk


def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else 132


def test_plans_match_the_table():
    with open(mk.OUT) as f:
        want = json.load(f)
    got = mk.rows()
    assert sorted(got) == sorted(want), "the recorded groups changed: regenerate the table"
    k = 2 if _sms() == 132 else 1      # digest index: with or without grid
    bad = [g for g, r in got.items() if mk.digest(r)[0] != want[g][0] or mk.digest(r)[k] != want[g][k]]
    assert not bad, f"{len(bad)} of {len(want)} plan groups differ; current plans:\n" + "\n".join(
        f"{r} grid={grid}" for g in bad[:5] for r, grid in got[g])
