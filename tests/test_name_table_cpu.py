"""The decode kernel's name table without a GPU: every struct-tag name and finish_reason value maps to itself, in any ASCII case
(with the upper-case flag the google map and finish_reason values use), and every one-byte variant of one maps to nothing."""
import pytest

from tests.name_table import build_harness, finish_names, hash_mul, lookup, schema_names, table_names

NONE = 0xFF


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    return build_harness(str(tmp_path_factory.mktemp("name_table")))


def test_names_map_to_themselves(exe):
    names = table_names()
    assert len(names) == len(set(names)) and {n for _, n in schema_names()} | set(finish_names()) == set(names)
    strings = [n.encode() for n in names] + [n.upper().encode() for n in names] + [n.title().encode() for n in names]
    mul, got = lookup(exe, strings)
    assert mul == hash_mul(names), "the Python restatement of the hash differs from build_tables"
    k = len(names)
    for i, n in enumerate(names):
        assert got[i] == (i, 0), n
        assert got[k + i] == (i, 1), n.upper()
        assert got[2 * k + i] == (i, int(n.title() != n)), n.title()


def one_byte_variants(n: bytes):
    """Substitutions (other than a letter's own case), deletions and insertions of one printable ASCII byte."""
    out = set()
    alphabet = [bytes([c]) for c in range(0x20, 0x7F)]
    for i in range(len(n)):
        out.add(n[:i] + n[i + 1:])
        for c in alphabet:
            if c.lower() != n[i:i + 1]:
                out.add(n[:i] + c + n[i + 1:])
    for i in range(len(n) + 1):
        for c in alphabet:
            out.add(n[:i] + c + n[i:])
    return sorted(out)


def test_one_byte_variants_miss(exe):
    names = table_names()
    folded = {n.encode() for n in names}
    strings = [v for n in names for v in one_byte_variants(n.encode()) if v.lower() not in folded and b"\\" not in v]
    assert len(strings) > 50000
    _, got = lookup(exe, strings)
    bad = [(s, g) for s, g in zip(strings, got) if g[0] != NONE]
    assert not bad, f"{len(bad)} variants match a name, first {bad[:5]}"


def test_empty_long_and_non_ascii_miss(exe):
    strings = [b"", b"a" * 20, b"finish_reason" + b"x" * 67, b"stop\x80", b"choice\xc5\xbf", b"to\xe2\x84\xaaen", b"\xc3\xa9"]
    _, got = lookup(exe, strings)
    assert all(g[0] == NONE for g in got), got
