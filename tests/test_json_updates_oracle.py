"""The JSON-updates reference (tests/json_updates_ref.cpp on the oracle) pinned by the reference's known answers
(crates/loro/tests/integration_test/detached_editing_test.rs:97-..., redact_test.rs:28-95) and by the invariants of every export on random
histories: per peer the ids cover exactly [start, end), op lengths add up, lamports never decrease, peers are indexed in
order of first use."""
import json
import random

from oracle import OracleDoc
from tests import json_updates_checks as jc
from tests import workloads


def test_detached_editing_known_answer():
    # peer 1 writes "Hello world!" (one change once stored), peer 2 inserts " alice!" at version {1: 5}, peer 1 then
    # prepends "Hi " on top of both: deps 4@0 and 11@0, 6@1, lamports 0 / 5 / 12, peers [1, 2]
    a = OracleDoc(1)
    t = a.get_text("text")
    a.text_insert(t, 0, "Hello")
    a.commit()
    first = a.export_updates()
    a.text_insert(t, 5, " world!")
    a.commit()
    b = OracleDoc(2)
    b.import_(first)
    b.text_insert(b.get_text("text"), 5, " alice!")
    b.commit()
    a.import_(b.export_updates())
    a.text_insert(t, 0, "Hi ")
    a.commit()
    doc = jc.oracle_doc([a.export_updates()])
    got = json.loads(jc.export_json_updates(doc))
    text = "cid:root-text:Text"
    assert got == {
        "schema_version": 1, "start_version": {}, "peers": ["1", "2"],
        "changes": [
            {"id": "0@0", "timestamp": 0, "deps": [], "lamport": 0, "msg": None,
             "ops": [{"container": text, "content": {"type": "insert", "pos": 0, "text": "Hello world!"}, "counter": 0}]},
            {"id": "0@1", "timestamp": 0, "deps": ["4@0"], "lamport": 5, "msg": None,
             "ops": [{"container": text, "content": {"type": "insert", "pos": 5, "text": " alice!"}, "counter": 0}]},
            {"id": "12@0", "timestamp": 0, "deps": ["11@0", "6@1"], "lamport": 12, "msg": None,
             "ops": [{"container": text, "content": {"type": "insert", "pos": 0, "text": "Hi "}, "counter": 12}]},
        ]}
    # without compression the ids carry the peers themselves; start_version lists the heads of the start version
    raw = json.loads(jc.export_json_updates(doc, {1: 12, 2: 7}, None, peer_compression=False))
    assert raw["peers"] is None and raw["start_version"] == {"1": 11, "2": 6}
    assert [c["id"] for c in raw["changes"]] == ["12@1"] and raw["changes"][0]["deps"] == ["11@1", "6@2"]
    # {1: 5, 2: 7} has 4@1 in the past of 6@2: the frontiers are 6@2 alone
    assert json.loads(jc.export_json_updates(doc, {1: 5, 2: 7}))["start_version"] == {"2": 6}


# redact_test.rs:28-95 before the redaction: the values the test inserted stand where the redacted text has nulls
REDACT_EXPECTED = """{
  "schema_version": 1,
  "start_version": {},
  "peers": [
    "1"
  ],
  "changes": [
    {
      "id": "0@0",
      "timestamp": 0,
      "deps": [],
      "lamport": 0,
      "msg": null,
      "ops": [
        {
          "container": "cid:root-map:Map",
          "content": {
            "type": "insert",
            "key": "key1",
            "value": "sensitive data"
          },
          "counter": 0
        },
        {
          "container": "cid:root-map:Map",
          "content": {
            "type": "insert",
            "key": "key2",
            "value": 42
          },
          "counter": 1
        },
        {
          "container": "cid:root-list:List",
          "content": {
            "type": "insert",
            "pos": 0,
            "value": [
              "secret info",
              true
            ]
          },
          "counter": 2
        }
      ]
    }
  ]
}"""


def redact_blob():
    """the document of redact_map_list_insertions: one change of peer 1 with two map inserts and two list inserts"""
    d = OracleDoc(1)
    m, lst = d.get_map("map"), d.get_list("list")
    d.map_set(m, "key1", "sensitive data")
    d.map_set(m, "key2", 42)
    d.list_insert(lst, 0, "secret info")
    d.list_insert(lst, 1, True)
    d.commit()
    return d.export_updates()


def test_redact_known_answer():
    doc = jc.oracle_doc([redact_blob()])
    text = jc.export_json_updates(doc)
    assert json.dumps(json.loads(text), indent=2, ensure_ascii=False) == REDACT_EXPECTED


def test_invariants_on_random_histories():
    rng = random.Random(1)
    for seed in range(6):
        blob = workloads.make_doc_history(8100 + seed, n_sites=2 + seed % 3, n_ops=150)[0]
        doc = jc.oracle_doc([blob])
        vv = doc.oplog_vv()
        for _ in range(6):
            s, e = jc.random_range(rng, vv)
            for pc in (True, False):
                jc.check_invariants(jc.export_json_updates(doc, s, e, pc), s, e, vv)
