"""The parts of tests/golden/engine_plans.json.gz the engine plans without a device: for every configuration of
tools/dump_engine_plans.py the parameter table, the weight blob size and the workspace size at each batch
(b200_ncsnpp_workspace_bytes plans dry).  tests/test_gpu_engine_plans.py checks the bound op tables."""
import json

import pytest

from tools import dump_engine_plans as D

PLANS = D.load()
CASES = D.cases()


def test_golden_covers_the_matrix():
  assert sorted(PLANS) == sorted(c['key'] for c in CASES)


@pytest.mark.parametrize('case', CASES, ids=[c['key'] for c in CASES])
def test_planned_sizes_match_golden(case):
  got = json.loads(json.dumps(D.planned_record(case)))
  want = PLANS[case['key']]
  assert got == {k: want[k] for k in got}
