"""The threshold arithmetic of tests/test_gpu_scale.py, checked with the oracle alone: every scale case, generated and
compacted on the CPU, still reaches the level its name promises (survivor, block and filter-block counts, the
straddling block, buckets, ticket rounds). A generator or oracle change that moves a case off its threshold fails here,
before any GPU time is spent. The case table and the levels are in tests/scale_cases.py."""
import pytest

import scale_cases as sc


@pytest.mark.parametrize("case_id", [c.id for c in sc.CASES])
def test_case_crosses_its_threshold(oracle, case_id):
    case = sc.BY_ID[case_id]
    _, inputs, exp, out = sc.run_oracle(case)
    assert out is not None
    assert exp.stats.num_input_records == sum(s.num_entries for s in inputs)
    sc.assert_crossed(case, sc.levels(case, inputs, exp, out))


def test_straddle_detection():
    """straddles() on hand-made block cuts: the first start of group 1 at offset SEG counts (also when the block before
    it started late in group 0), one at SEG - 1 does not, and a group without a block start is passed over."""
    G, S = sc.GROUP, sc.SEG
    assert sc.straddles([G + S, 10]) == [1]
    assert sc.straddles([G + S - 1, 10]) == []
    assert sc.straddles([G - 5, S + 5, 10]) == [1]
    assert sc.straddles([G + 10, S, 10]) == []
    assert sc.straddles([2 * G + S, 10]) == [2]
