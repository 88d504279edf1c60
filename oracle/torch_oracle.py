"""float64 oracle of the TF-IDF, Jaccard and dense-cosine scores, in torch, on any device.  TEST INFRASTRUCTURE ONLY.

The same math as :func:`oracle.tfidf_oracle.score_matrix_closed_form` (DESIGN §3), restated so that an H100 can score
a block of queries against millions of rows in well under a second.  It never looks inside an index: its inputs are
the raw CSR of the rows (``indptr``, ``ids``, ``tf``) and of the queries (plus ``oov``, the tf² sum of each query's
out-of-vocabulary features), as the host featuriser produces them, and optionally a live-row mask, per-row labels and
global statistics (``df``, ``N``).  It computes df itself, by counting over the live rows, unless ``df`` is given.
Nothing here imports ``kakveda_b200``.

Identical rows get bit-identical scores: every row's entries are put in ascending feature order once, and every row
sum (norm, dot product, correction) adds its terms in that order, one row position at a time (no sparse library
whose summation order could depend on where a row sits in memory).  The exact-tie checks of the tests rely on it.
"""
from __future__ import annotations

import math
from typing import Optional, Tuple

import torch

F64 = torch.float64


def _t(a, device, dtype=None):
    t = torch.as_tensor(a, device=device)
    return t.to(dtype) if dtype is not None else t


def _canonical(indptr: torch.Tensor, ids: torch.Tensor, vals: torch.Tensor, width: int):
    """(row, pos, ids, vals) of a CSR with every row's entries in ascending id order; pos = position inside the row."""
    n = len(indptr) - 1
    lens = indptr[1:] - indptr[:-1]
    row = torch.repeat_interleave(torch.arange(n, device=indptr.device), lens)
    order = torch.argsort(row * width + ids, stable=True)
    row, ids, vals = row[order], ids[order], vals[order]
    pos = torch.arange(len(row), device=indptr.device) - indptr[:-1][row]
    return row, pos, ids, vals


def _rowsum_by_position(n: int, row: torch.Tensor, pos: torch.Tensor, terms, width: int = 0) -> torch.Tensor:
    """out[r] = the sum of row r's terms, added in position order starting from 0.0.  ``terms(sel)`` gives the terms
    of the entries ``sel`` ([len(sel)] when ``width`` is 0, else [len(sel), width]); it is called once per position, so
    that the terms of all entries never exist at once."""
    out = torch.zeros((n, width) if width else (n,), dtype=F64, device=row.device)
    if len(pos) == 0:
        return out
    by_pos = torch.argsort(pos, stable=True)
    counts = torch.bincount(pos).tolist()
    start = 0
    for c in counts:           # within one position every row occurs at most once: one add per output element
        sel = by_pos[start:start + c]
        out.index_add_(0, row[sel], terms(sel))
        start += c
    return out


class SparseOracle:
    """Rows of a TF-IDF or Jaccard index, for :meth:`tfidf_scores` and :meth:`jaccard_counts` of query blocks.

    ``vocab_size``: feature ids are below it.  ``live``: bool [N], False for a deleted row (scores -inf; not counted in
    N or df).  ``labels``: int [N], matched against the per-query labels of a filtered block (other rows: -inf).
    ``df`` / ``n_global``: global statistics replacing the ones counted over the live rows."""

    def __init__(self, indptr, ids, tf, vocab_size: int, device="cpu", live=None, labels=None, df=None,
                 n_global: Optional[int] = None):
        dev = torch.device(device)
        self.device, self.V = dev, int(vocab_size)
        indptr = _t(indptr, dev, torch.int64)
        self.n = len(indptr) - 1
        self.row, self.pos, self.ids, self.tf = _canonical(indptr, _t(ids, dev, torch.int64), _t(tf, dev, F64), self.V)
        self.lens = (indptr[1:] - indptr[:-1]).to(F64)
        self.live = None if live is None else _t(live, dev, torch.bool)
        self.labels = None if labels is None else _t(labels, dev, torch.int64)
        if df is None:
            keep = torch.ones_like(self.row, dtype=torch.bool) if self.live is None else self.live[self.row]
            self.df = torch.bincount(self.ids[keep], minlength=self.V)[: self.V].to(F64)
        else:
            self.df = _t(df, dev, F64)[: self.V]
        self.N = float(n_global if n_global is not None else (self.n if self.live is None else int(self.live.sum())))
        self._norms = {}
        self._slot = torch.full((self.V + 1,), -1, dtype=torch.int64, device=dev)

    # -- statistics -------------------------------------------------------------------------------------------------
    def _weights(self, mode: int):
        """(a, d, idf0², idf²_rows) per feature: query weight a, correction d = a - idf_row², and the row idf²."""
        n, df = self.N, self.df
        if mode == 0:   # the reference's refit: the query is one more document
            idf_b = torch.log((n + 2.0) / (df + 1.0)) + 1.0
            idf_q = torch.log((n + 2.0) / (df + 2.0)) + 1.0
            return idf_q ** 2, idf_q ** 2 - idf_b ** 2, (math.log((n + 2.0) / 2.0) + 1.0) ** 2, idf_b ** 2
        idf = torch.log((n + 1.0) / (df + 1.0)) + 1.0   # mode 2: fitted on the corpus alone
        w = torch.where(df > 0, idf ** 2, torch.zeros_like(idf))
        return w, torch.zeros_like(w), 0.0, w

    def _row_norms(self, mode: int) -> torch.Tensor:
        if mode not in self._norms:
            rowidf2 = self._weights(mode)[3]
            w = self.tf * self.tf * rowidf2[self.ids]
            self._norms[mode] = _rowsum_by_position(self.n, self.row, self.pos, lambda e: w[e])
        return self._norms[mode]

    # -- a query block restricted to its features -----------------------------------------------------------------
    def _block(self, q_indptr, q_ids, q_tf, keep_feature):
        """(feats [F], Wtf [F+1, B] query tf, member [F+1, B], entries (row, pos, slot, tf) of the rows restricted
        to the block's features).  Row F of the [F+1, B] matrices is zero."""
        dev = self.device
        q_indptr = _t(q_indptr, dev, torch.int64)
        B = len(q_indptr) - 1
        qi = _t(q_ids, dev, torch.int64)
        qt = _t(q_tf, dev, F64)
        qrow = torch.repeat_interleave(torch.arange(B, device=dev), q_indptr[1:] - q_indptr[:-1])
        ok = qi < self.V
        ok[ok.clone()] = keep_feature(qi[ok])
        qi, qt, qrow = qi[ok], qt[ok], qrow[ok]
        feats = torch.unique(qi)
        F = len(feats)
        slot_of = torch.searchsorted(feats, qi)
        Wtf = torch.zeros((F + 1, B), dtype=F64, device=dev)
        Wtf.index_put_((slot_of, qrow), qt, accumulate=True)   # a feature listed twice in one query adds its tf
        member = (Wtf > 0).to(F64)
        self._slot[feats] = torch.arange(F, device=dev)
        slot = self._slot[self.ids]
        self._slot[feats] = -1
        sel = slot >= 0
        row, tf, slot = self.row[sel], self.tf[sel], slot[sel]
        # position inside the restricted row, in canonical order
        starts = torch.zeros(self.n + 1, dtype=torch.int64, device=dev)
        starts[1:] = torch.cumsum(torch.bincount(row, minlength=self.n), 0)
        pos = torch.arange(len(row), device=dev) - starts[:-1][row]
        return feats, Wtf, member, (row, pos, slot, tf)

    def _mask(self, s: torch.Tensor, query_labels) -> torch.Tensor:
        if self.live is not None:
            s[:, ~self.live] = -math.inf
        if query_labels is not None:
            ql = _t(query_labels, self.device, torch.int64)
            s.masked_fill_((ql[:, None] >= 0) & (self.labels[None, :] != ql[:, None]), -math.inf)
        return s

    def tfidf_scores(self, q_indptr, q_ids, q_tf, q_oov, mode: int = 0, query_labels=None) -> torch.Tensor:
        """[B, N] float64 TF-IDF cosine of a block of queries.  mode 0: the reference's refit (idf of the query's
        features with df + 1 and N + 2); mode 2: fitted on the corpus (features with df = 0 and out-of-vocabulary
        ones are ignored).  -inf for deleted rows and rows a query's label excludes."""
        a, d, idf0sq, _ = self._weights(mode)
        keep = (lambda f: torch.ones_like(f, dtype=torch.bool)) if mode == 0 else (lambda f: self.df[f] > 0)
        feats, Wtf, member, (row, pos, slot, tf) = self._block(q_indptr, q_ids, q_tf, keep)
        F = len(feats)
        af = torch.zeros(F + 1, dtype=F64, device=self.device)
        df_ = torch.zeros(F + 1, dtype=F64, device=self.device)
        af[:F], df_[:F] = a[feats], d[feats]
        nq = ((Wtf * Wtf) * af[:, None]).sum(0)
        if mode == 0:
            nq = nq + _t(q_oov, self.device, F64) * idf0sq
        W, Dm, B = Wtf * af[:, None], member * df_[:, None], Wtf.shape[1]
        dot = _rowsum_by_position(self.n, row, pos, lambda e: W[slot[e]] * tf[e, None], B)
        corr = _rowsum_by_position(self.n, row, pos, lambda e: Dm[slot[e]] * (tf[e] * tf[e])[:, None], B)
        den = nq[None, :] * (self._row_norms(mode)[:, None] + corr)
        ok = (den > 0) & (dot != 0)
        s = torch.where(ok, dot / torch.sqrt(torch.where(ok, den, torch.ones_like(den))), torch.zeros_like(den)).T
        return self._mask(s.contiguous(), query_labels)

    def jaccard_counts(self, q_indptr, q_ids, q_oov=None) -> Tuple[torch.Tensor, torch.Tensor]:
        """Exact (inter, union) float64 [B, N] of token sets (0/1 sums, exact below 2^53).  Query ids must be distinct;
        ids outside the vocabulary only count towards |q|, as do ``q_oov`` more of them per query."""
        q_indptr = _t(q_indptr, self.device, torch.int64)
        q_ids = _t(q_ids, self.device, torch.int64)
        ones = torch.ones(len(q_ids), dtype=F64, device=self.device)
        _, _, member, (row, pos, slot, _) = self._block(q_indptr, q_ids, ones, lambda f: torch.ones_like(f, dtype=torch.bool))
        inter = _rowsum_by_position(self.n, row, pos, lambda e: member[slot[e]], member.shape[1]).T.contiguous()
        qlen = (q_indptr[1:] - q_indptr[:-1]).to(F64)
        if q_oov is not None:
            qlen = qlen + _t(q_oov, self.device, F64)
        return inter, qlen[:, None] + self.lens[None, :] - inter

    def jaccard_scores(self, q_indptr, q_ids, q_oov=None) -> torch.Tensor:
        """[B, N] float64 inter / union (0 / 0 -> 0)."""
        inter, union = self.jaccard_counts(q_indptr, q_ids, q_oov)
        return torch.where(union > 0, inter / union.clamp(min=1), torch.zeros_like(inter))


def bf16_round(x) -> torch.Tensor:
    """float -> bfloat16 (round to nearest even) -> float64, the values the dense kernel computes with."""
    return torch.as_tensor(x).to(torch.float32).to(torch.bfloat16).to(F64)


def dense_cosine(Q, C) -> torch.Tensor:
    """[Q, N] float64 cosine of the bf16-rounded rows (torch tensors on one device, or arrays); zero vectors score 0."""
    q64, c64 = bf16_round(Q), bf16_round(C)
    qn = torch.sqrt((q64 * q64).sum(1))
    cn = torch.sqrt((c64 * c64).sum(1))
    den = qn[:, None] * cn[None, :]
    d = q64 @ c64.T
    return torch.where(den > 0, d / torch.where(den > 0, den, torch.ones_like(den)), torch.zeros_like(den))
