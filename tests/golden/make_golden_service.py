"""Golden vectors for the resident-GFKB service layer (kakveda_b200/store.py), made by RUNNING THE UNMODIFIED
REFERENCE handlers ``/failures/upsert`` and ``/failures/match`` (services/gfkb/app.py:79-147) through FastAPI's
TestClient (needs a checkout of the reference, its directory in KAKVEDA_REFERENCE):

    python tests/golden/make_golden_service.py

A seeded request stream (new failures, repeats of earlier (failure_type, signature_text) pairs from other apps,
evolving resolution / root_cause) is replayed; after every few upserts a set of match requests is issued.  The file
keeps the requests, the record each upsert returned (timestamps dropped: they are wall-clock) and the matches.
Also: corpus-fit TF-IDF all-pairs goldens (sklearn fit(corpus)/transform) for the self-join mode.
"""
from __future__ import annotations

import json
import pathlib
import random
import sys
import tempfile
import os
from pathlib import Path

HERE = Path(__file__).resolve().parent
REPO = HERE.parent.parent
REF = Path(os.environ["KAKVEDA_REFERENCE"])
sys.path.insert(0, str(REPO))
sys.path.insert(0, str(REF))

import numpy as np  # noqa: E402

from kakveda_b200 import synth  # noqa: E402
from oracle import tfidf_oracle as O  # noqa: E402


def dump(name, obj):
    p = HERE / name
    p.write_text(json.dumps(obj, ensure_ascii=False, separators=(",", ":")) + "\n", encoding="utf-8")
    print(f"wrote {p} ({p.stat().st_size} bytes)")


def strip(rec):
    return {k: v for k, v in rec.items() if k not in ("created_at", "updated_at")}


def main():
    _orig_mkdir = pathlib.Path.mkdir

    def _safe_mkdir(self, *a, **kw):  # the module mkdirs /app/data at import (app.py:23-24)
        if str(self).startswith("/app"):
            return None
        return _orig_mkdir(self, *a, **kw)

    pathlib.Path.mkdir = _safe_mkdir
    import services.gfkb.app as gfkb_app
    pathlib.Path.mkdir = _orig_mkdir
    from fastapi.testclient import TestClient

    rng = random.Random(20260921)
    texts = synth.corpus(60)
    types = ["HALLUCINATION_CITATION", "TOOL_MISUSE", "TIMEOUT"]
    apps = ["app-a", "app-b", "app-c", "app-d"]
    steps = []
    with tempfile.TemporaryDirectory() as td:
        f = Path(td) / "failures.jsonl"
        gfkb_app.FAILURES_FILE = f
        client = TestClient(gfkb_app.app)
        issued = []
        for i in range(90):
            if issued and rng.random() < 0.45:
                ft, st = rng.choice(issued)  # repeat -> new version
            else:
                ft, st = rng.choice(types), rng.choice(texts)
            issued.append((ft, st))
            req = {"failure_type": ft, "signature_text": st, "app_id": rng.choice(apps),
                   "context_signature": {"k": rng.randrange(5)} if rng.random() < 0.7 else {},
                   "impact_severity": rng.choice(["low", "medium", "high"]),
                   "root_cause": rng.choice([None, "rc-%d" % i]), "resolution": rng.choice([None, "fix-%d" % i])}
            resp = client.post("/failures/upsert", json=req)
            assert resp.status_code == 200, resp.text
            body = resp.json()
            step = {"upsert": req, "created": body["created"], "failure": strip(body["failure"])}
            if i % 6 == 5 or i == 89:
                ms = []
                qs = [rng.choice(texts) for _ in range(3)] + [rng.choice(issued)[1], synth.queries(1, 60)[0]]
                for q in qs:
                    ft = rng.choice([None, None] + types)
                    body = {"signature_text": q}
                    if ft:
                        body["failure_type"] = ft
                    m = client.post("/failures/match", json=body)
                    assert m.status_code == 200, m.text
                    ms.append({"signature_text": q, "failure_type": ft, "matches": m.json()["matches"]})
                step["matches"] = ms
            steps.append(step)
        final = [strip(json.loads(l)) for l in f.read_text().splitlines() if l.strip()]
    dump("service_upsert.json", {"source": "services/gfkb/app.py:79-147 via TestClient", "steps": steps, "final_records": final})

    # corpus-fit TF-IDF (sklearn fit(corpus).transform(queries)) and its all-pairs top-k, seeded synthetic rows
    n, k = 400, 8
    corpus = synth.corpus(n)
    S = O.corpus_fit_scores(corpus, corpus)
    rows, vals = O.allpairs_topk(S, k)
    qs = synth.queries(6, n)
    Sq = O.corpus_fit_scores(qs, corpus)
    dump("corpus_fit.json", {"n": n, "k": k, "allpairs_rows": rows.tolist(), "allpairs_scores": vals.tolist(),
                             "row_sums": S.sum(axis=1).tolist(), "query_scores": Sq.tolist(),
                             "source": "sklearn TfidfVectorizer(ngram_range=(1,2)).fit(corpus) / transform + cosine_similarity"})


if __name__ == "__main__":
    main()
