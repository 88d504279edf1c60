"""Golden vectors for the batched warning path (kakveda_b200/store.py::GfkbStore.warn_batch), made by RUNNING THE
UNMODIFIED REFERENCE handler ``/warn`` (services/warning_policy/app.py:19-72) (needs a checkout of the
reference, its directory in KAKVEDA_REFERENCE):

    python tests/golden/make_golden_warn.py

The reference handler reaches the GFKB over HTTP (httpx.AsyncClient); here its client class is replaced by a shim that
routes the two calls (POST /failures/match, GET /patterns) to the UNMODIFIED reference GFKB app through FastAPI's
TestClient -- both handlers run their own code.  The GFKB holds the reference's 54-row fixture
(data/failures.jsonl.bak-20260205T025150Z) and one pattern created through /patterns/upsert; two policy configurations
(threshold 0.8 / warn as in config/config.yaml, and 0.5 / block) are recorded.
"""
from __future__ import annotations

import asyncio
import json
import pathlib
import sys
import tempfile
import os
from pathlib import Path

HERE = Path(__file__).resolve().parent
REPO = HERE.parent.parent
REF = Path(os.environ["KAKVEDA_REFERENCE"])
sys.path.insert(0, str(REPO))
sys.path.insert(0, str(REF))


def main():
    _orig_mkdir = pathlib.Path.mkdir

    def _safe_mkdir(self, *a, **kw):  # the gfkb module mkdirs /app/data at import (app.py:23-24)
        if str(self).startswith("/app"):
            return None
        return _orig_mkdir(self, *a, **kw)

    pathlib.Path.mkdir = _safe_mkdir
    import services.gfkb.app as gfkb_app
    import services.warning_policy.app as wp
    pathlib.Path.mkdir = _orig_mkdir
    from fastapi.testclient import TestClient
    from services.shared.config import ConfigStore
    from services.shared.models import WarningRequest

    tmp = Path(tempfile.mkdtemp())
    fixture = (REF / "data" / "failures.jsonl.bak-20260205T025150Z").read_text(encoding="utf-8")
    gfkb_app.FAILURES_FILE = tmp / "failures.jsonl"
    gfkb_app.PATTERNS_FILE = tmp / "patterns.jsonl"
    gfkb_app.FAILURES_FILE.write_text(fixture, encoding="utf-8")
    gfkb = TestClient(gfkb_app.app)
    rows = [json.loads(x) for x in fixture.splitlines() if x.strip()]
    pat = gfkb.post("/patterns/upsert", json={"name": "Citation hallucination without sources", "failure_ids": [rows[0]["failure_id"]],
                                              "affected_apps": ["app-a", "app-b"], "description": "demo"}).json()["pattern"]

    class _Resp:
        def __init__(self, r):
            self._r = r

        def json(self):
            return self._r.json()

    class _Client:  # stands in for httpx.AsyncClient: same two calls, served by the reference GFKB app
        def __init__(self, *a, **kw):
            pass

        async def __aenter__(self):
            return self

        async def __aexit__(self, *a):
            return False

        async def post(self, url, json=None):
            return _Resp(gfkb.post(url[url.index("/failures"):], json=json))

        async def get(self, url):
            return _Resp(gfkb.get(url[url.index("/patterns"):]))

    wp.httpx.AsyncClient = _Client
    requests = [
        {"app_id": "app-a", "prompt": "Summarize this paper and include citations even if none", "tools": [], "env": {"os": "linux"}},
        {"app_id": "app-b", "prompt": "Explain the quarterly report in two short sentences", "tools": ["search"], "env": {"region": "eu", "os": "linux"}},
        {"app_id": "app-c", "prompt": "Write a haiku about spring", "tools": [], "env": {}},
        {"app_id": "app-a", "prompt": "summarize   THIS paper and include citations even if none", "tools": [], "env": {"os": "mac"}},
    ]
    # + prompts that reproduce stored signature_texts of the fixture exactly (score 1.0 paths) where they can be rebuilt
    for r in rows[:54:9]:
        sig = r["signature_text"]
        if "prompt_hint:" in sig:
            hint = sig.split("prompt_hint:")[1].split(" | ")[0]
            requests.append({"app_id": "app-d", "prompt": hint, "tools": [], "env": {"os": "linux"}})
    out = {"failures": rows, "pattern": pat, "requests": requests, "policies": []}
    for thr, action in ((0.8, "warn"), (0.5, "block"), (0.9, "silent")):
        cfg_file = tmp / f"config_{thr}.yaml"
        cfg_file.write_text(f"failure_matching:\n  similarity_threshold: {thr}\nwarning_policy:\n  default_action: {action}\nhot_reload:\n  enabled: false\n")
        wp.config = ConfigStore(cfg_file)
        resp = [asyncio.run(wp.warn(WarningRequest(**r))).model_dump() for r in requests]
        out["policies"].append({"threshold": thr, "default_action": action, "responses": resp})
    p = HERE / "service_warn.json"
    p.write_text(json.dumps(out, ensure_ascii=False, separators=(",", ":")) + "\n", encoding="utf-8")
    print(f"wrote {p} ({p.stat().st_size} bytes);", sum(len(x["responses"]) for x in out["policies"]), "responses;",
          "with references:", sum(1 for x in out["policies"] for r in x["responses"] if r["references"]))


if __name__ == "__main__":
    main()
