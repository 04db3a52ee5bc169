"""CPU: the digest verdict of tests/util.py. A run equal to its oracle passes; each rule fails on a corruption of one field of
one connection, and on nothing else; skip exempts exactly the connections it lists."""
import re

import numpy as np
import pytest

from inference_gateway_b200 import _abi as A
from oracle import orc
from tests.util import DIGEST_FIELDS, RULES, assert_digest_parity, parity_faults

LIVE, TERMINATED = 1, 3
# name: (the rule it breaks, the connection it changes, the field: a digest field, "carry" or "seg_flags", what is added to
# the field or, for seg_flags, the bits flipped)
CORRUPTIONS = {**{f: ("digests", LIVE, f, 1) for f in DIGEST_FIELDS}, "inexact": ("inexact", LIVE, "inexact", 1),
               "carry": ("carry", LIVE, "carry", 1), "terminated_early": ("termination", LIVE, "seg_flags", A.SEG_TERMINATED),
               "not_terminated": ("termination", TERMINATED, "seg_flags", A.SEG_TERMINATED),
               "dead": ("seg_flags", LIVE, "seg_flags", A.SEG_DEAD),
               "line_too_long": ("seg_flags", LIVE, "seg_flags", A.SEG_LINE_TOO_LONG),
               "deferred": ("seg_flags", LIVE, "seg_flags", A.SEG_DEFERRED),
               "finished_live": ("finished", LIVE, "seg_flags", A.SEG_FINISHED)}


def clean():
    """(run, oracle) that agree: connections 0-2 live with carried tails, 3-5 terminated, 5 also FINISHED. A terminated
    connection's carry is not the oracle's tail (the tail is dropped at the end of the stream)."""
    od = orc.new_digests(6)
    for k, f in enumerate(DIGEST_FIELDS):
        od[f] = np.arange(6) * 10 + k + 1
    oterm = np.array([0, 0, 0, 1, 1, 1], dtype=np.uint8)
    otail = np.array([5, 0, 17, 0, 0, 0], dtype=np.uint32)
    flags = np.array([0, 0, 0, 1, 1, 1], dtype=np.uint32) * A.SEG_TERMINATED
    flags[5] |= A.SEG_FINISHED
    return (od.copy(), np.array([5, 0, 17, 0, 9, 0], dtype=np.uint32), flags), (od, oterm, otail)


def test_a_run_equal_to_the_oracle_passes():
    got, oracle = clean()
    assert parity_faults(got, oracle) == {}
    assert assert_digest_parity(got, None, None, "clean", oracle=oracle) is oracle[0]


@pytest.mark.parametrize("name", list(CORRUPTIONS))
def test_each_rule_fails_on_its_own_corruption(name):
    rule, conn, field, change = CORRUPTIONS[name]
    got, oracle = clean()
    if field == "seg_flags":
        got[2][conn] ^= change
    else:
        (got[1] if field == "carry" else got[0][field])[conn] += change
    faults = parity_faults(got, oracle)
    assert list(faults) == [rule] and faults[rule].tolist() == [conn]
    with pytest.raises(AssertionError, match=re.escape(RULES[rule])):
        assert_digest_parity(got, None, None, name, oracle=oracle)
    assert_digest_parity(got, None, None, name, oracle=oracle, skip=[conn])


def test_skip_exempts_exactly_the_listed_connections():
    got, oracle = clean()
    got[0]["recs_h"][[0, 2, 4]] += 1
    assert parity_faults(got, oracle, skip=[0, 4])["digests"].tolist() == [2]
    with pytest.raises(AssertionError, match=r"first \[2\]"):
        assert_digest_parity(got, None, None, "skip", oracle=oracle, skip=[0, 4])
    assert_digest_parity(got, None, None, "skip", oracle=oracle, skip=[0, 2, 4])
