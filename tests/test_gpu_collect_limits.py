"""The collect pass of the default exec mode (exec_matches) at its phrase limit, on both sides and both codecs, against the reference's
exec_query: an OR of 32 two-term phrases over 32 distinct terms is answered bit for bit, hits included; a 33rd phrase node is refused with
the planner's message, and the context answers the next call."""
import numpy as np
import pytest

import trinity_b200 as tb
from matchutil import doc_corpus
from test_gpu_matched_terms import CODECS, IDS, Side

pytestmark = pytest.mark.gpu
NAMES = [f"t{i + 1}" for i in range(32)]
PAIRS = [(NAMES[i], NAMES[(i + 1) % 32]) for i in range(32)] + [(NAMES[0], NAMES[2])]  # 32 distinct phrases over 32 terms, then a 33rd


def phrases(n):
    return " OR ".join(f'"{a} {b}"' for a, b in PAIRS[:n])


@pytest.mark.parametrize("codec", CODECS, ids=IDS)
def test_32_phrase_nodes_and_33_refused(codec):
    rng = np.random.default_rng(41)
    lists, _ = doc_corpus(rng, 3000, 32, (3, 40))
    s = Side(codec, lists, 3000, NAMES)
    q32, q33 = phrases(32), phrases(33)
    nodes = tb.parse_query(q32, s.tdict)
    assert sum(int(x["kind"]) == tb.NODE_PHRASE for x in nodes) == 32
    assert len(set(int(x["term"]) for x in nodes if int(x["kind"]) == tb.NODE_TERM)) == 32
    cases = [(q32, 0, 0)] + [(f'"{a} {b}"', 0, 0) for a, b in PAIRS[:32:8]]
    res = s.check(cases)
    assert res.hits.size > 0
    # the docIDs ran on the step program, and the matched terms and hits came from the collect pass (k_collect_count / k_collect_write)
    assert s.gpu.last_routes().tolist() == [tb.ROUTE_STEPS] * len(cases)
    assert res.chunks >= 1 and res.count_ms > 0 and res.write_ms > 0
    for i in range(len(cases)):  # every phrase of the OR matches some documents, and misses others
        assert 0 < len(s.ref.exec(cases[i][0])) < 3000
    with pytest.raises(tb.TrinityError, match="rc=-7: .*query 1: the default exec mode takes at most 32 phrase nodes per query"):
        s.gpu.exec_matches([nodes, tb.parse_query(q33, s.tdict)])
    s.check([(q32, 0, 0)])
