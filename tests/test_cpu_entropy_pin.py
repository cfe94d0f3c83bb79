"""The split schedules tests/test_gpu_entropy_pin.py runs K6's entropy variant on, checked without a GPU.

aa_linear_logprob_fwd keeps three floats of `partial` per (row, vocabulary split), its entropy variant four (the
entropy sum t rides along), and both lower the split count until n * splits * floats fits `partial_floats`
(linear_logprob.cu make_schedule).  So one `partial` buffer can give the two launches different split counts, and
with them a different merge order of the row statistics.  The pin runs every lm_head pin case (FWD_CASES) at three
budgets:
  * 'wide4': room for every split the schedule wants at four floats per split;
  * 'none':  no `partial` at all (one CTA sweeps the whole vocabulary);
  * '<kind>3': the case's own kind counted at three floats per split -- what a caller that sizes `partial` for the plain
    launch hands the entropy launch.
Here the schedule is restated at 3 and 4 floats per split for a 132-SM H100, every case is shown to reach the schedule
its note names, and the budgets at which the two launches split differently are listed.
"""
from __future__ import annotations

import pytest

from test_gpu_lm_head_tiles import BM, BN, FWD_CASES, _fwd_case_id, schedule

SMS = 132  # H100 SXM


def k6_budgets(case, sms=SMS):
    """-> {budget name: partial_floats} of one FWD_CASES entry (the own-kind budget is left out when it is 'none')."""
    n, _, _, kind, _ = case
    own = {'none': 0, 'wide': n * sms * 3, 'two': n * 2 * 3}[kind]
    out = {'wide4': n * sms * 4, 'none': 0}
    if kind != 'none':
        out[f'{kind}3'] = own
    return out


def k6_splits(case, budget, per_split, sms=SMS):
    """(splits, tiles per split) of a launch with `per_split` floats per (row, split) at the named budget."""
    n, _, V, _, _ = case
    pf = k6_budgets(case, sms)[budget]
    splits, tps, _ = schedule(n, V, pf > 0, pf, per_split, sms)
    return splits, tps


K6_PARAMS = [(c, b) for c in FWD_CASES for b in k6_budgets(c)]
K6_IDS = [f'{_fwd_case_id(c)}-{b}' for c, b in K6_PARAMS]
# the budgets at which the plain launch (3 floats per split) and the entropy launch (4) pick different split counts
SPLIT_COUNTS_DIFFER = {'129x320x777-two-two3', '1000x128x5000-two-two3'}


def test_split_counts_differ_only_where_listed():
    differ = {i for i, (c, b) in zip(K6_IDS, K6_PARAMS) if k6_splits(c, b, 3) != k6_splits(c, b, 4)}
    assert differ == SPLIT_COUNTS_DIFFER, differ
    for i, (c, b) in zip(K6_IDS, K6_PARAMS):
        if i in SPLIT_COUNTS_DIFFER:  # the plain launch merges two splits, the entropy launch runs unsplit
            assert k6_splits(c, b, 3)[0] == 2 and k6_splits(c, b, 4)[0] == 1, i


def test_wide4_gives_the_entropy_launch_every_split():
    """'wide4' lets the entropy launch split as far as the schedule wants: the count of a launch without a budget."""
    for c in FWD_CASES:
        n, _, V, _, _ = c
        assert k6_splits(c, 'wide4', 4) == schedule(n, V, True, -1, 4, SMS)[:2], _fwd_case_id(c)
        assert k6_splits(c, 'none', 4)[0] == 1


def _note_holds(case):
    """The schedule each FWD_CASES note names, at the case's own budget (3 floats, the lm_head pin) and at 'wide4'."""
    n, H, V, kind, _ = case
    units, all_tiles, k_blocks = -(-n // BM), -(-V // BN), H // 64
    own = 'none' if kind == 'none' else f'{kind}3'
    s3, tps3 = k6_splits(case, own, 3)
    s4 = k6_splits(case, 'wide4', 4)[0]
    last = all_tiles - (s3 - 1) * tps3  # tiles of the last split
    cid = _fwd_case_id(case)
    notes = {
        '1x64x1-wide': lambda: V == 1 and s3 == s4 == 1 and k_blocks == 1,
        # split 1 is the last tile alone, which holds one column; 3 k-blocks fill less than the 4-stage ring
        '63x192x257-wide': lambda: s3 == s4 == 2 and tps3 == 1 and V - BN == 1 and k_blocks == 3,
        '129x320x777-none': lambda: s3 == 1 and V % BN == 9,
        '200x64x513-wide': lambda: s3 == s4 == 3 and tps3 == 1 and V - 2 * BN == 1 and k_blocks == 1,
        '129x320x777-two': lambda: (s3 == 2 and k6_splits(case, 'two3', 4)[0] == 1
                                    and schedule(n, V, True, -1, 3, SMS)[0] > 2),
        # 132 // 3 = 44 splits wanted, 42 after dropping empty ones
        '300x4096x32064-wide': lambda: units < SMS // 8 and s3 == s4 == 42,
        '300x4096x32064-none': lambda: s3 == 1,
        '2100x256x32064-wide': lambda: units >= SMS // 8 and 6 <= s3 <= 16 and s3 == s4,
        # the splits do not divide the vocabulary evenly: the last one is short and ends in the one-column last tile
        '260x4096x128257-wide': lambda: s3 == s4 > 1 and 0 < last < tps3 and V % BN == 1,
        # 16 splits wanted (10 after dropping empty ones), 2 fit at 3 floats, 1 at 4
        '1000x128x5000-two': lambda: (SMS // units == 16 and schedule(n, V, True, -1, 3, SMS)[0] == 10 and s3 == 2
                                      and k6_splits(case, 'two3', 4)[0] == 1),
    }
    return notes[cid]()


@pytest.mark.parametrize('case', FWD_CASES, ids=[_fwd_case_id(c) for c in FWD_CASES])
def test_each_case_reaches_the_schedule_its_note_names(case):
    assert _note_holds(case), (_fwd_case_id(case), case[4])


def test_restated_schedule_matches_hand_counts():
    """Hand-checked: 1000 rows are 8 row units (< 132 / 8), so 132 // 8 = 16 splits over the 20 vocabulary tiles of
    V = 5000, 2 tiles each -> 10 splits; 6000 floats hold 2 splits at 3 floats per row and split, 1 at 4."""
    assert schedule(1000, 5000, True, -1, 3, SMS)[:2] == (10, 2)
    assert schedule(1000, 5000, True, 6000, 3, SMS)[:2] == (2, 10)
    assert schedule(1000, 5000, True, 6000, 4, SMS)[:2] == (1, 20)
    assert schedule(1000, 5000, True, 8000, 4, SMS)[:2] == (2, 10)
