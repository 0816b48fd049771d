#!/usr/bin/env python3
"""Transcribe TestOrchestrateConcurrentMoves (orchestrate_test.go:452-1047) into
tests/golden/orchestrate_concurrency_cases.json, with the Go-literal parser of make_fixtures.py plus the two things
this table needs: the AssignPartitionsFunc field type, and the fmt.Errorf(...) value of the "empty assignPartitions
callback" case (which has no expectation and is skipped).

Per case: model, maxConcurrentMoves, nodesAll, begMap, endMap, expNode, skipCallbacks, expConcurrentMovesCount,
the expected partitions and states (the test sorts both before comparing) and the expected ops (in pick order: the
test compares them unsorted).  No reference source is copied, only the table's data.  Only needed when
regenerating:  python tests/golden/make_schedule_fixtures.py [path to the reference tree]"""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_fixtures as mf  # noqa: E402

mf.NAMED["AssignPartitionsFunc"] = ("ptr", ("basic", "func"))   # a func value: nil unless set


class Parser(mf.Parser):
    def parse_value(self, want=None):
        if self.peek() == ("id", "fmt") and self.peek(1)[1] == "." and self.peek(2)[1] == "Errorf":
            self.i += 3
            self.expect("(")
            msg = self.parse_value()
            while self.accept("+"):
                msg += self.parse_value()
            self.expect(")")
            return {"error": msg}
        return super().parse_value(want)


def concurrency_cases(toks):
    env = mf.package_vars(toks, ("mrPartitionModel",))
    body = mf.func_body_tokens(toks, "TestOrchestrateConcurrentMoves")
    p = Parser(body, env)
    while p.peek()[1] != "tests":                 # options := OrchestratorOptions{}
        p.next()
    p.next(); p.next()
    out = []
    for idx, c in enumerate(p.parse_value()):
        if c["skip"]:
            continue
        out.append({"index": idx, "label": c["label"], "model": mf.model_json(c["partitionModel"]),
                    "maxConcurrentMoves": c["maxConcurrentMoves"], "nodesAll": c["nodesAll"],
                    "begMap": mf.pmap_json(c["begMap"]), "endMap": mf.pmap_json(c["endMap"]),
                    "expNode": c["expNode"], "skipCallbacks": c["skipCallbacks"],
                    "expConcurrentMovesCount": c["expConcurrentMovesCount"],
                    "expMovePartitions": c["expMovePartitions"], "expMoveStates": c["expMoveStates"],
                    "expMoveOps": c["expMoveOps"]})
    return out


def main():
    toks = mf.tokenize(open(os.path.join(mf.REF, "orchestrate_test.go")).read())
    cases = concurrency_cases(toks)
    with open(os.path.join(mf.OUT, "orchestrate_concurrency_cases.json"), "w") as f:
        json.dump(cases, f, indent=1, sort_keys=True)
    print("orchestrate concurrency cases: %d" % len(cases))


if __name__ == "__main__":
    main()
