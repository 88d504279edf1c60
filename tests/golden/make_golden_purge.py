"""Golden vectors for the app purge of the resident GFKB (``GfkbStore.purge_apps``), made by RUNNING THE UNMODIFIED
REFERENCE: the gfkb handlers ``/failures/upsert`` and ``/failures/match`` (services/gfkb/app.py:79-147) through
FastAPI's TestClient, and the dashboard's ``_purge_jsonl_apps`` (services/dashboard/app.py:330-375) on the same
failures.jsonl.  Needs a checkout of the reference, its directory in KAKVEDA_REFERENCE:

    python tests/golden/make_golden_purge.py

Importing services.dashboard.app needs packages the generator does not (sqlalchemy, the dashboard's own modules), so
only the ``_purge_jsonl_apps`` function definition is compiled out of the file (``ast``), with ``json`` and ``Path``
as its globals.  A seeded upsert stream (new failures, repeats of earlier (failure_type, signature_text) pairs from
other apps) is replayed; the file is purged twice, of different apps, with match requests before and after each
purge and further upserts between them -- new ids after a purge follow the reference's F-%04d of len(records) + 1,
collisions with surviving ids included.  The fixture keeps the requests, the purge arguments and counts, the surviving
lines and the responses (timestamps dropped: they are wall-clock).
"""
from __future__ import annotations

import __future__
import ast
import json
import os
import pathlib
import random
import sys
import tempfile
from pathlib import Path

HERE = Path(__file__).resolve().parent
REPO = HERE.parent.parent
REF = Path(os.environ["KAKVEDA_REFERENCE"])
sys.path.insert(0, str(REPO))
sys.path.insert(0, str(REF))

from kakveda_b200 import synth  # noqa: E402


def dump(name, obj):
    p = HERE / name
    p.write_text(json.dumps(obj, ensure_ascii=False, separators=(",", ":")) + "\n", encoding="utf-8")
    print(f"wrote {p} ({p.stat().st_size} bytes)")


def strip(rec):
    return {k: v for k, v in rec.items() if k not in ("created_at", "updated_at")}


def reference_purge():
    """``_purge_jsonl_apps`` compiled out of services/dashboard/app.py as it stands."""
    src_path = REF / "services" / "dashboard" / "app.py"
    tree = ast.parse(src_path.read_text(encoding="utf-8"))
    fn = next(n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name == "_purge_jsonl_apps")
    mod = ast.Module(body=[fn], type_ignores=[])
    scope = {"json": json, "Path": Path}
    exec(compile(mod, str(src_path), "exec", flags=__future__.annotations.compiler_flag, dont_inherit=True), scope)
    return scope["_purge_jsonl_apps"]


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

    purge = reference_purge()
    rng = random.Random(20261016)
    texts = synth.corpus(50)
    types = ["HALLUCINATION_CITATION", "TOOL_MISUSE", "TIMEOUT"]
    apps = ["app-a", "app-b", "app-c", "app-d", "demo-1", "demo-2"]
    steps = []
    with tempfile.TemporaryDirectory() as td:
        f = Path(td) / "failures.jsonl"
        gfkb_app.FAILURES_FILE = f
        client = TestClient(gfkb_app.app)
        issued = []

        def upsert(i):
            if issued and rng.random() < 0.5:
                ft, st = rng.choice(issued)  # repeat -> new version, possibly from another app
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
            steps.append({"upsert": req, "created": body["created"], "failure": strip(body["failure"])})

        def matches():
            ms = []
            qs = [rng.choice(texts) for _ in range(4)] + [rng.choice(issued)[1], synth.queries(1, 50)[0]]
            for q in qs:
                ft = rng.choice([None, None] + types)
                body = {"signature_text": q}
                if ft:
                    body["failure_type"] = ft
                m = client.post("/failures/match", json=body)
                assert m.status_code == 200, m.text
                ms.append({"signature_text": q, "failure_type": ft, "matches": m.json()["matches"]})
            steps.append({"matches": ms})

        def purge_step(app_ids):
            before = [strip(json.loads(l)) for l in f.read_text(encoding="utf-8").splitlines() if l.strip()]
            counts = purge(f, set(app_ids))
            after = [strip(json.loads(l)) for l in f.read_text(encoding="utf-8").splitlines() if l.strip()]
            steps.append({"purge": sorted(app_ids), "counts": counts, "lines_before": before, "lines": after})

        for i in range(70):
            upsert(i)
            if i % 10 == 9:
                matches()
        purge_step(["demo-1", "demo-2"])
        matches()
        for i in range(70, 100):
            upsert(i)
            if i % 10 == 9:
                matches()
        purge_step(["app-a"])
        matches()
        for i in range(100, 115):
            upsert(i)
        matches()
    dump("purge.json", {"source": "services/gfkb/app.py:79-147 via TestClient + services/dashboard/app.py:330-375",
                        "steps": steps})


if __name__ == "__main__":
    main()
