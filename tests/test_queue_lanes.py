"""The verify queue's side lanes, the batch lane (hs_queue_batch) and the explain lane (hs_queue_explain), share one state type and one
set of functions in hs_engine.cu: one site takes a lane request's arena region, one function polls the lanes' completion words, and
one function configures either lane."""
import re

from test_launch_sites import _code


def _body(code, head):
    """The body of the function whose definition starts with `head`."""
    m = re.search(re.escape(head) + r"[^;{]*\{", code)
    assert m, head
    depth, i = 1, m.end()
    while depth:
        depth += {"{": 1, "}": -1}.get(code[i], 0)
        i += 1
    return code[m.end():i - 1]


def test_arena_regions_are_taken_at_one_site_for_both_lanes():
    code = _code()
    takes = re.findall(r"\.take\(", code)
    # the ring's preimage arena (hs_queue_submit_msgs) and the side lanes' arenas
    assert len(takes) == 2, takes
    assert len(re.findall(r"\.take\(", _body(code, "static int lane_submit("))) == 1


def test_lane_completion_words_are_polled_in_one_function():
    # a host read of word [1] of a region's tail, its completion word (k_queue_explain and k_batch_done write it)
    poll = r"const volatile uint32_t\s*\*\s*>\([^;]*o_tail\s*\)\s*\[\s*1\s*\]"
    code = _code()
    assert len(re.findall(poll, code)) == 1, re.findall(poll, code)
    assert re.search(poll, _body(code, "static void lane_complete("))


def test_both_lane_entry_points_call_the_one_configure_function():
    code = _code()
    assert len(re.findall(r"static int lane_configure\(", code)) == 1
    for entry in ("int hs_queue_batch(", "int hs_queue_explain("):
        assert "lane_configure(" in _body(code, entry), entry
