"""Plan identity: for every configuration of tools/dump_engine_plans.py the engine binds exactly the plan recorded in
tests/golden/engine_plans.json.gz - the same ops in the same order with the same labels, kinds, flops and algorithmic bytes,
the same parameter table, weight and workspace sizes, launches per forward and PC loop sizes."""
import json

import pytest
import torch

from tools import dump_engine_plans as D

PLANS = D.load()
CASES = D.cases()


@pytest.mark.gpu
@pytest.mark.parametrize('case', CASES, ids=[c['key'] for c in CASES])
def test_bound_plan_matches_golden(case):
  got = json.loads(json.dumps(D.bound_record(case, torch.device('cuda:0'))))
  want = PLANS[case['key']]
  for i, (g, w) in enumerate(zip(got['ops'], want['ops'])):
    assert g == w, f'op {i}: {g} != {w}'
  assert len(got['ops']) == len(want['ops'])
  assert {k: v for k, v in got.items() if k != 'ops'} == {k: v for k, v in want.items() if k != 'ops'}
