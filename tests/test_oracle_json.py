"""CPU: pins the oracle's encoding/json restatement against an independent model (tests/go_model.py: CPython's
json for syntax + a typed decode written from the Go documentation) on hand-written and mutated documents."""
import numpy as np
import pytest

from inference_gateway_b200 import synth
from oracle import orc
from tests import go_model
from tests.corpus import (STRING_EVENTS, STRING_LENGTHS, TRICKY, mutate, string_alignment_docs, string_offsets,
                          template_near_misses)
from tests.util import chunk_to_dict


def test_tricky_documents():
    for d in TRICKY:
        d = d.replace(b"\n", b" ")
        assert chunk_to_dict(orc.unmarshal(d)) == go_model.unmarshal(d), d


@pytest.mark.parametrize("seed", [0, 1])
def test_mutation_fuzz(seed):
    rng = np.random.default_rng(seed)
    streams, _ = synth.make_config("C4", n_streams=40)
    docs = [ev[6:] for b, _, _ in streams for ev in b.split(b"\n\n") if ev.startswith(b"data: {")] + TRICKY
    n_ok = 0
    for _ in range(6000):
        d = mutate(rng, docs[int(rng.integers(0, len(docs)))])
        a = chunk_to_dict(orc.unmarshal(d))
        assert a == go_model.unmarshal(d), d
        assert orc.json_valid(d) == go_model.parse(d)[0], d
        n_ok += a["json_ok"]
    assert 1000 < n_ok < 5900      # the corpus exercises both outcomes


def test_string_alignment_corpus():
    """The GPU occupancy tests take the oracle as truth on this corpus: pin it here first, on every document."""
    docs = string_alignment_docs()
    assert docs == string_alignment_docs()                        # deterministic
    assert len(docs) == len(STRING_EVENTS) * sum(len(string_offsets(n)) for n in STRING_LENGTHS)
    n_ok = 0
    for d in docs:
        a = chunk_to_dict(orc.unmarshal(d))
        assert a == go_model.unmarshal(d), d[:200]
        n_ok += a["json_ok"]
    assert 0 < n_ok < len(docs)


def test_template_near_miss_corpus():
    canon, miss = template_near_misses()
    assert (canon, miss) == template_near_misses()
    for d in canon:
        assert chunk_to_dict(orc.unmarshal(d))["json_ok"], d
    n_ok = 0
    for d in canon + miss:
        a = chunk_to_dict(orc.unmarshal(d))
        assert a == go_model.unmarshal(d), d
        n_ok += a["json_ok"]
    assert len(canon) < n_ok < len(canon) + len(miss)


def test_trim_space_matches_unicode_isspace():
    # unicode.IsSpace (Go): White_Space property
    go_space = ["\t", "\n", "\v", "\f", "\r", " ", "", " ", " ", " ", " ", " ", " ",
                "　"] + [chr(c) for c in range(0x2000, 0x200B)]
    for ws in go_space:
        s = (ws + "a" + ws + ws).encode()
        assert orc.trim_space(s) == b"a", repr(ws)
    for not_ws in ["​", "᠎", "﻿", "⁠", "\x1c", "\x1f", "\x00"]:     # not White_Space for Go
        s = (not_ws + "a").encode()
        assert orc.trim_space(s) == s, repr(not_ws)
    assert orc.trim_space(b" \xe2\x80 a\xe2\x80") == b"\xe2\x80 a\xe2\x80"               # truncated sequences stay
    assert orc.trim_space(b"") == b"" and orc.trim_space(b" \t\r\n") == b""


def test_number_rules():
    ok = lambda s: orc.unmarshal(b'{"created":%s}' % s).json_ok
    assert ok(b"0") and ok(b"-0") and ok(b"9223372036854775807") and ok(b"-9223372036854775808")
    assert not ok(b"9223372036854775808") and not ok(b"1.0") and not ok(b"1e3") and not ok(b'"1"') and not ok(b"true")
    lp = lambda s: orc.unmarshal(b'{"choices":[{"logprobs":{"content":[{"logprob":%s}]}}]}' % s).json_ok
    assert lp(b"-9999.0") and lp(b"3.4028234e38") and lp(b"3.40282356e38") and lp(b"1e-999")
    assert not lp(b"3.4028236e38") and not lp(b"1e39") and not lp(b"-4e38")
    assert lp(b"340282356779733661637539395458142568447") and not lp(b"340282356779733661637539395458142568448")


def test_depth_limit_rule_matches_independent_scan():
    """The oracle's restatement of the nesting limit (orc_json_scan at 128 levels) against a bracket count up to CPython's
    first syntax error (tests/go_model.py::depth_limited), on the nesting corpus and on every corpus document."""
    from tests.corpus import nesting_docs
    docs = nesting_docs()
    n_limited = 0
    for name, d, twin in docs:
        lim = orc.json_scan(d, orc.DEPTH_LIMIT) == orc.JSON_DEPTH
        assert lim == go_model.depth_limited(d), name
        assert not go_model.depth_limited(twin), name
        n_limited += lim
    for d in TRICKY:
        assert (orc.json_scan(d, orc.DEPTH_LIMIT) == orc.JSON_DEPTH) == go_model.depth_limited(d), d
    names = {n for n, _, _ in docs}
    assert len(docs) > 1000 and 200 < n_limited < len(docs) - 200
    # the shape of the rule at its edges
    assert {n: orc.json_scan(d, orc.DEPTH_LIMIT) for n, d, _ in docs if n.startswith("top-arr")} == \
        {"top-arr-d127": 0, "top-arr-d128": 0, "top-arr-d129": 2, "top-arr-d130": 2}
    by = {n: orc.json_scan(d, orc.DEPTH_LIMIT) for n, d, _ in docs}
    assert by["syntax_before-d130"] == orc.JSON_SYNTAX and by["syntax_after-d130"] == orc.JSON_DEPTH
    assert by["mismatch_open-alt-k64"] == orc.JSON_SYNTAX and by["mismatch_open-alt-k129"] == orc.JSON_DEPTH
    assert by["in_string-d130"] == orc.JSON_OK and "mismatch_deep-rnd-k65" in names
