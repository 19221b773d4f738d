"""The stream table (tests/stream_cases.py) against include/centerpose_b200.h: every entry point that takes a stream is
held on a side stream by tests/test_streams_gpu.py or exempted with a reason, so a new one cannot arrive untested."""
import ctypes

from centerpose_b200 import _lib
from tests.stream_cases import EXEMPT, HELD, covered, stream_entry_points


def _header():
    with open(_lib.HEADER) as f:
        return f.read()


def test_every_stream_entry_point_is_held_or_exempt():
    declared = stream_entry_points(_header())
    missing = declared - covered() - set(EXEMPT)
    assert not missing, "entry points with a stream and no case in tests/stream_cases.py: %s" % sorted(missing)


def test_table_names_only_declared_entry_points():
    declared = stream_entry_points(_header())
    stale = (covered() | set(EXEMPT)) - declared
    assert not stale, "tests/stream_cases.py names entry points the header does not declare with a stream: %s" % sorted(stale)
    assert not covered() & set(EXEMPT), sorted(covered() & set(EXEMPT))
    assert all(EXEMPT.values()) and all(HELD.values())


def test_parser_finds_a_new_declaration():
    text = _header() + "\nint cpb200_new_thing(const float *x, int n,\n                     void *stream);\n" \
                       "int cpb200_no_stream(const float *x);\n"
    found = stream_entry_points(text)
    assert "new_thing" in found and "no_stream" not in found
    assert found - {"new_thing"} == stream_entry_points(_header())
    # every declared stream parameter is the prototype's last, as _lib.launch appends it
    for name in stream_entry_points(_header()):
        assert _lib.signatures()["cpb200_" + name][1][-1] is ctypes.c_void_p, name
