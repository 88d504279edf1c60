"""Binary sidecar of ``failures.jsonl`` (SURVEY.md section 8(f) rank 4).

The reference re-reads, re-validates and re-tokenises the whole JSONL on every request
(services/gfkb/app.py:38-56,81; similarity.py:17-18).  A resident store only pays that at start-up -- and with a
sidecar not even then: the file keeps what featurisation produced (the vocabulary's 128-bit feature keys in id order
and the CSR of every row) together with a digest of the ``signature_text`` column it was built from.  ``load`` returns
the arrays only if the digest still matches the first ``n`` records of the JSONL (the GFKB is append-only,
app.py:132,146, so a longer file is a valid extension: the new rows are featurised on top); anything else is treated
as stale and ignored.  The scan layout itself (text sort, stream, summaries) is rebuilt by ``finalize`` -- host work
that needs the global statistics anyway.

Format: one ``.npz`` (NumPy, uncompressed): ``keys`` uint64[V,2], ``indptr`` int64[n+1], ``ids`` uint32[nnz],
``tf`` uint16[nnz], ``meta`` = [format version, n, nnz, V], ``digest`` = sha256 over the signature_texts.
"""
from __future__ import annotations

import hashlib
from pathlib import Path
from typing import Optional, Sequence, Tuple

import numpy as np

from .similarity import ArrayBatch, FeatureBatch, Vocabulary

FORMAT_VERSION = 1


def digest(signature_texts: Sequence[str]) -> bytes:
    h = hashlib.sha256()
    for t in signature_texts:
        b = t.encode("utf-8")
        h.update(len(b).to_bytes(8, "little"))
        h.update(b)
    return h.digest()


def save(path: Path, vocab: Vocabulary, batch, signature_texts: Sequence[str]) -> None:
    """``batch``: the FeatureBatch / ArrayBatch of exactly ``signature_texts`` (featurised with ``vocab``)."""
    if batch.n != len(signature_texts):
        raise ValueError("sidecar.save: batch and texts differ in length")
    if batch.tf.size and int(batch.tf.max()) > 65535:
        raise ValueError("sidecar.save: term frequency above 65535")
    keys = vocab.export_keys()
    tmp = Path(str(path) + ".tmp.npz")
    np.savez(tmp, keys=keys, indptr=np.asarray(batch.indptr, dtype=np.int64), ids=np.asarray(batch.ids, dtype=np.uint32),
             tf=np.asarray(batch.tf).astype(np.uint16), meta=np.array([FORMAT_VERSION, batch.n, len(batch.ids), len(keys)], dtype=np.int64),
             digest=np.frombuffer(digest(signature_texts), dtype=np.uint8))
    tmp.replace(path)


def load(path: Path, signature_texts: Sequence[str]) -> Optional[Tuple[Vocabulary, ArrayBatch, int]]:
    """(vocabulary, CSR of the first n rows, n) if the sidecar describes a prefix of ``signature_texts``, else None."""
    path = Path(path)
    if not path.exists():
        return None
    try:
        with np.load(path) as z:
            meta = z["meta"]
            if int(meta[0]) != FORMAT_VERSION:
                return None
            n, nnz, v = int(meta[1]), int(meta[2]), int(meta[3])
            if n > len(signature_texts) or bytes(z["digest"].tobytes()) != digest(signature_texts[:n]):
                return None
            keys, indptr, ids, tf = z["keys"], z["indptr"], z["ids"], z["tf"]
            if keys.shape != (v, 2) or len(indptr) != n + 1 or len(ids) != nnz or len(tf) != nnz or (nnz and int(ids.max()) >= v):
                return None
            return Vocabulary.from_keys(keys), ArrayBatch(indptr, ids, tf.astype(np.uint32)), n
    except Exception:  # unreadable / truncated / foreign file: the sidecar is only a cache
        return None


def load_arrays(path: Path) -> Optional[Tuple[ArrayBatch, int]]:
    """(CSR of the rows, n) as the file holds them, without the digest check of ``load`` -- for a writer that knows
    which rows it saved (``GfkbStore`` rewriting its own sidecar after a purge); None if missing or unreadable."""
    path = Path(path)
    if not path.exists():
        return None
    try:
        with np.load(path) as z:
            meta = z["meta"]
            if int(meta[0]) != FORMAT_VERSION:
                return None
            n, nnz = int(meta[1]), int(meta[2])
            indptr, ids, tf = z["indptr"], z["ids"], z["tf"]
            if len(indptr) != n + 1 or len(ids) != nnz or len(tf) != nnz:
                return None
            return ArrayBatch(indptr, ids, tf.astype(np.uint32)), n
    except Exception:  # unreadable / truncated / foreign file: the sidecar is only a cache
        return None
