"""TLC's -dump on the host: the command line's -dump forms and the dot writer (kafka_specification_b200/dump.py)."""
import io

import numpy as np
import pytest

from kafka_specification_b200 import dump
from kafka_specification_b200.dump import split_dump_args
from kafka_specification_b200.runtime import EDGE_DTYPE
from kafka_specification_b200.tlc2 import parse_args


@pytest.mark.parametrize("argv,rest,path,dot,options", [
    (["-dump", "states", "Spec"], ["Spec"], "states.dump", False, []),
    (["-dump", "out.dump", "Spec"], ["Spec"], "out.dump", False, []),
    (["-deadlock", "-dump", "d/x", "-config", "S.cfg", "Spec"], ["-deadlock", "-config", "S.cfg", "Spec"], "d/x.dump",
     False, []),
    (["-dump", "dot", "g", "Spec"], ["Spec"], "g.dot", True, []),
    (["-dump", "dot,actionlabels", "g.dot", "Spec"], ["Spec"], "g.dot", True, ["actionlabels"]),
    (["-dump", "dot,actionlabels,colorize,snapshot", "g", "-workers", "1", "Spec"], ["-workers", "1", "Spec"], "g.dot",
     True, ["actionlabels", "colorize", "snapshot"]),
    (["Spec", "-dump", "dot,colorize", "g"], ["Spec"], "g.dot", True, ["colorize"]),
    # a state dump whose name ends in .dot is still a state dump
    (["-dump", "g.dot", "Spec"], ["Spec"], "g.dot.dump", False, []),
])
def test_dump_forms_leave_spec_positional(argv, rest, path, dot, options):
    got_rest, req = split_dump_args(argv)
    assert got_rest == rest
    assert (req.path, req.dot, req.options) == (path, dot, options)
    assert parse_args(got_rest).spec == "Spec"


def test_no_dump_is_untouched():
    assert split_dump_args(["-deadlock", "Spec"]) == (["-deadlock", "Spec"], None)


@pytest.mark.parametrize("argv", [["-dump"], ["Spec", "-dump", "dot"], ["-dump", "dot,bogus", "g", "Spec"],
                                  ["-dump", "a", "-dump", "b", "Spec"]])
def test_malformed_dump_is_refused(argv):
    with pytest.raises(ValueError):
        split_dump_args(argv)


def test_cli_refuses_malformed_dump_with_spec_error_code():
    from kafka_specification_b200 import tlc2
    assert tlc2.main(["-dump", "dot,bogus", "g", "Spec"]) == tlc2.EXIT_ERROR_SPEC


def edges(rows):
    e = np.zeros(len(rows), dtype=EDGE_DTYPE)
    for i, (src_fp, dst_fp, action) in enumerate(rows):
        e[i]["src_fp"], e[i]["dst_fp"], e[i]["action"] = src_fp, dst_fp, action
    return e


BIG = 2 ** 64 - 5          # prints as -5


def graph(**kw):
    f = io.StringIO()
    texts = ['/\\ x = 1\n/\\ s = "a\\b"', "/\\ x = 2", "/\\ x = 3"]
    e = edges([(1, 2, 0), (2, BIG, 1), (1, 2, 0), (2, 2, 1), (1, 2, 1)])
    n = dump.write_dot(f, np.array([1, 2, BIG], dtype=np.uint64), texts, 1, e, ["Inc", "Stay"], **kw)
    return f.getvalue(), n


def test_dot_layout():
    text, n = graph()
    lines = text.splitlines()
    assert lines[0] == "strict digraph DiskGraph {"
    assert lines[-1] == "}"
    assert n == {"nodes": 3, "edges": 4}
    # escaping: backslash, quote, newline; the initial state is filled, the others are not
    assert '1 [label="/\\\\ x = 1\\n/\\\\ s = \\"a\\\\b\\"",style = filled]' in lines
    assert '2 [label="/\\\\ x = 2"]' in lines
    assert '-5 [label="/\\\\ x = 3"]' in lines
    # edges deduplicated, self-loops kept, ids signed, ordered by (src, dst, action)
    assert [l for l in lines if "->" in l] == ["1 -> 2;", "1 -> 2;", "2 -> 2;", "2 -> -5;"]
    assert "legend" not in text and "label=\"Inc\"" not in text


def test_dot_labels_and_colours():
    text, _ = graph(actionlabels=True, colorize=True)
    lines = text.splitlines()
    assert lines[1] == 'edge [colorscheme="paired12"]'
    assert [l for l in lines if "->" in l] == [
        '1 -> 2 [label="Inc",color="1",fontcolor="1"];', '1 -> 2 [label="Stay",color="2",fontcolor="2"];',
        '2 -> 2 [label="Stay",color="2",fontcolor="2"];', '2 -> -5 [label="Stay",color="2",fontcolor="2"];']
    assert 'Inc [label="Inc",fillcolor=1]' in lines and 'Stay [label="Stay",fillcolor=2]' in lines
    assert lines.index('Inc [label="Inc",fillcolor=1]') > lines.index('subgraph cluster_legend {graph[style=bold];'
                                                                      'label = "Next State Actions" style="solid"')
    labels, _ = graph(actionlabels=True)
    assert '1 -> 2 [label="Inc"];' in labels and "fontcolor" not in labels


def test_dot_is_deterministic_in_the_edge_order():
    a, _ = graph(actionlabels=True)
    f = io.StringIO()
    texts = ['/\\ x = 1\n/\\ s = "a\\b"', "/\\ x = 2", "/\\ x = 3"]
    e = edges([(1, 2, 1), (2, 2, 1), (2, BIG, 1), (1, 2, 0)])
    dump.write_dot(f, np.array([1, 2, BIG], dtype=np.uint64), texts, 1, e, ["Inc", "Stay"], actionlabels=True)
    assert f.getvalue() == a


def test_state_blocks_and_row_order():
    f = io.StringIO()
    assert dump.write_states(f, ["/\\ x = 1", "/\\ x = 2"], 3) == 2
    assert f.getvalue() == "State 3:\n/\\ x = 1\n\nState 4:\n/\\ x = 2\n\n"
    rows = np.array([[2, 0], [1, 5], [1, 3]], dtype=np.uint64)
    assert dump.sorted_rows(rows).tolist() == [[1, 3], [1, 5], [2, 0]]
