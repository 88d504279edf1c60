"""Generate the golden vectors under tests/golden/ by RUNNING THE UNMODIFIED REFERENCE.

Needs a checkout of the reference (its directory in KAKVEDA_REFERENCE); the tests only read the JSON output:

    python tests/golden/make_golden.py

Everything numerical in the JSON files comes from ``services.shared.similarity.SimilarityEngine``
(services/shared/similarity.py:14-20), ``services.shared.fingerprint`` (fingerprint.py:51-71) and the
GFKB handler ``services.gfkb.app.match`` (services/gfkb/app.py:79-102) imported from
the reference checkout; inputs are either the reference's own test / fixture data or seeded synthetic rows
from ``kakveda_b200.synth`` (regenerated, and checksum-verified, at test time).
"""
from __future__ import annotations

import hashlib
import json
import sys
import os
from pathlib import Path

HERE = Path(__file__).resolve().parent
REPO = HERE.parent.parent
REF = Path(os.environ["KAKVEDA_REFERENCE"])
sys.path.insert(0, str(REPO))
sys.path.insert(0, str(REF))

import numpy as np  # noqa: E402

from services.shared.similarity import SimilarityEngine  # noqa: E402  (the reference)
from services.shared import fingerprint as ref_fp  # noqa: E402

from kakveda_b200 import synth  # noqa: E402


def sha(texts) -> str:
    h = hashlib.sha256()
    for t in texts:
        h.update(t.encode("utf-8"))
        h.update(b"\n")
    return h.hexdigest()


def dump(name: str, obj) -> None:
    p = HERE / name
    p.write_text(json.dumps(obj, ensure_ascii=False, indent=None, separators=(",", ":")) + "\n", encoding="utf-8")
    print(f"wrote {p} ({p.stat().st_size} bytes)")


def topk(scores, k):
    order = sorted(range(len(scores)), key=lambda i: scores[i], reverse=True)[:k]
    return order, [scores[i] for i in order]


def main() -> None:
    eng = SimilarityEngine()

    # 1. the reference's own unit test inputs (tests/test_similarity.py:4-12)
    corpus = [
        "prompt: summarize and add references | tools: | env_keys:os",
        "prompt: write python code | tools: | env_keys:os",
    ]
    query = "prompt: summarize this and include citations | tools: | env_keys:os"
    dump("ref_test_similarity.json", {"source": "tests/test_similarity.py:4-12", "query": query, "corpus": corpus,
                                      "scores": eng.score(query, corpus)})

    # 2. the 54-row fixture data/failures.jsonl.bak-20260205T025150Z
    rows = [json.loads(l) for l in (REF / "data/failures.jsonl.bak-20260205T025150Z").read_text().splitlines() if l.strip()]
    records = [{k: r[k] for k in ("failure_id", "version", "failure_type", "resolution", "signature_text")} for r in rows]
    fx_corpus = [r["signature_text"] for r in records]
    demo = [  # scripts/demo_client.py:45-48,81 style payloads
        ("Summarize this paper and include citations even if none", [], {"os": "linux"}),
        ("Explain research paper and add references.", [], {"os": "linux"}),
        ("Short answer with citations", ["search"], {"os": "linux", "region": "eu"}),
        ("Write python code to sort a list", [], {"os": "linux"}),
    ]
    fx_queries = [ref_fp.signature_text(*d) for d in demo] + [fx_corpus[20], fx_corpus[0], "", "zz"]
    fx = {"source": "data/failures.jsonl.bak-20260205T025150Z", "records": records, "queries": fx_queries,
          "scores": [eng.score(q, fx_corpus) for q in fx_queries]}
    # the handler itself, through FastAPI's TestClient (services/gfkb/app.py:79-102)
    try:
        import tempfile
        from fastapi.testclient import TestClient
        import pathlib
        _orig_mkdir = pathlib.Path.mkdir

        def _safe_mkdir(self, *a, **kw):  # the module mkdirs /app/data at import (app.py:23-24)
            if str(self).startswith("/app"):
                return None
            return _orig_mkdir(self, *a, **kw)

        pathlib.Path.mkdir = _safe_mkdir
        import services.gfkb.app as gfkb_app
        pathlib.Path.mkdir = _orig_mkdir
        with tempfile.TemporaryDirectory() as td:
            f = Path(td) / "failures.jsonl"
            f.write_text("\n".join(json.dumps(r) for r in rows) + "\n")
            gfkb_app.FAILURES_FILE = f
            client = TestClient(gfkb_app.app)
            fx["match"] = []
            for q in fx_queries[:6]:
                for ft in (None, "HALLUCINATION_CITATION", "OTHER_TYPE"):
                    body = {"signature_text": q}
                    if ft:
                        body["failure_type"] = ft
                    resp = client.post("/failures/match", json=body)
                    assert resp.status_code == 200, resp.text
                    fx["match"].append({"signature_text": q, "failure_type": ft, "matches": resp.json()["matches"]})
    except Exception as e:  # pragma: no cover
        print("WARNING: gfkb.match goldens skipped:", e)
    dump("fixture54.json", fx)

    # 3. hand-written edge cases (unicode, tf > 1, empty rows, out-of-corpus query tokens ...)
    edge_corpus = [
        "alpha beta gamma delta",
        "alpha alpha alpha beta",
        "",
        "a b c",                       # no token of length >= 2
        "Alpha BETA Gamma",            # case folding
        "İstanbul ŞEHİR güzel straße STRASSE",
        "数据库 连接 失败 timeout timeout",
        "snake_case token_1 42 4x x4 __",
        "alpha beta gamma delta",       # exact duplicate of row 0
        "naïve café naïve café naïve",
        "tok " * 40 + "end",           # tf = 40 (> 31: overflow path of the scan layout)
        "beta gamma",
    ]
    edge_queries = ["alpha beta", "ALPHA  beta\tbeta", "unseen words only", "", "a", "İSTANBUL şehir", "数据库 timeout",
                    "tok tok end", "naïve café", "alpha beta gamma delta", "x4 4x 42 snake_case", "beta gamma delta alpha"]
    edge = {"corpus": edge_corpus, "queries": edge_queries, "scores": [eng.score(q, edge_corpus) for q in edge_queries]}
    # sklearn raises for an all-empty vocabulary
    try:
        eng.score("a", ["b", ""])
        edge["empty_vocab_raises"] = False
    except ValueError as e:
        edge["empty_vocab_raises"] = True
        edge["empty_vocab_message"] = str(e)
    dump("edge_cases.json", edge)

    # 4. seeded synthetic rows, small: every score
    n, q = 300, 12
    sc = synth.corpus(n)
    sq = synth.queries(q, n)
    dump("synthetic_small.json", {"n": n, "q": q, "corpus_seed": synth.CORPUS_SEED, "query_seed": synth.QUERY_SEED,
                                  "corpus_sha256": sha(sc), "queries_sha256": sha(sq),
                                  "scores": [eng.score(x, sc) for x in sq]})

    # 5. BASELINE cfg1: N=1000, Q=128 -- top-16 per query + row sums; full vectors for 8 queries
    n, q, k = 1000, 128, 16
    sc = synth.corpus(n)
    sq = synth.queries(q, n)
    full = [eng.score(x, sc) for x in sq]
    tk = [topk(s, k) for s in full]
    dump("synthetic_cfg1.json", {"n": n, "q": q, "k": k, "corpus_sha256": sha(sc), "queries_sha256": sha(sq),
                                 "topk_rows": [t[0] for t in tk], "topk_scores": [t[1] for t in tk],
                                 "score_sums": [float(np.sum(s)) for s in full], "full_first8": full[:8]})

    # 6. signature_text / fingerprint (fingerprint.py:51-71) on hand-written and synthetic inputs
    cases = [
        ("Summarize this paper and include citations even if none", ["search", "search", "sql"], {"os": 1, "region": 2}),
        ("  Explain   the\tReport\nwith REFERENCES  ", [], {}),
        ("tl;dr of the summary please", ["b", "a"], {"z": 0, "a": 0}),
        ("Describe sources; even if not provided include a bibliography " + "x" * 100, ["t"], {"k": None}),
        ("", [], {"os": "linux"}),
        ("Ünïcödé prompt with citations", ["tool"], {"env": 1}),
    ]
    sig = [{"prompt": p, "tools": t, "env_keys": sorted(e.keys()), "signature_text": ref_fp.signature_text(p, t, e),
            "fingerprint": ref_fp.fingerprint(p, t, e), "normalized": ref_fp.normalize_prompt(p)} for p, t, e in cases]
    # synthetic rows must be exactly what the reference's signature_text builds from their parts
    checked = 0
    for row in synth.corpus(2000):
        parts = row.split(" | ")
        hint = parts[1][len("prompt_hint:"):]
        if len(hint) >= 80:
            continue  # truncated hint: the full prompt (which drives the tags) is not recoverable
        tools = [t for t in parts[2][len("tools:"):].split(",") if t]
        env = {k: 1 for k in parts[3][len("env_keys:"):].split(",") if k}
        assert ref_fp.signature_text(hint, tools, env) == row, (row, ref_fp.signature_text(hint, tools, env))
        checked += 1
    print(f"synthetic rows checked against reference signature_text: {checked}")
    dump("signature_text.json", {"cases": sig, "synthetic_rows_checked": checked})


if __name__ == "__main__":
    main()
