"""CPU design study for the bound kernel's tile-local second-class (F2) dictionary (DESIGN.md sections 4 and 5): how
many distinct F2 features does a 128-query bound tile hold, how many (query, feature) incidences does a dictionary of
KT tensor-core columns cover, and how long would a per-warp loop over the rest run (the largest number of uncovered
features among a warp's 32 queries; KT = 0 is the per-query loop the dictionary replaced).  The bound kernel uses
KT = 256; its epilogue still loops over the uncovered features, and a warp whose queries have none skips that loop.

Approximations: feature classes are taken by document frequency over the sampled corpus (the index uses chunk frequency
over text-sorted 32-row chunks -- the same ranking up to ties); queries are text-sorted exactly as kv_query_upload
does.  Run:  python profiles/r2_sim_tile_f2_dictionary.py [rows] [queries]
"""
import sys
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from kakveda_b200 import synth  # noqa: E402
from kakveda_b200.similarity import Vocabulary  # noqa: E402

NF, NF2, TILE, Q2CAP = 256, 1024, 128, 24


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 1_000_000
    q = int(sys.argv[2]) if len(sys.argv) > 2 else 100_000
    buf, off = synth.signatures_packed(synth.CORPUS_SEED, 0, n)
    v = Vocabulary()
    fb = v.featurize_packed(buf, off, 0, grow=True)
    V = len(v)
    df = np.bincount(fb.ids, minlength=V)
    universal = df == n
    rank = np.argsort(-np.where(universal, -1, df), kind="stable")
    f1 = set(rank[:NF].tolist())
    f2 = np.zeros(V + 1, dtype=bool)
    f2[rank[NF:NF + NF2]] = True
    print(f"rows {n}  vocabulary {V}  universal {int(universal.sum())}  df of the F2 class: {df[rank[NF]]} .. {df[rank[NF + NF2 - 1]]}")
    fb.close()
    qb, qo = synth.signatures_packed(synth.QUERY_SEED, 0, q, dup_of_seed=synth.CORPUS_SEED, dup_rows=n)
    qf = v.featurize_packed(qb, qo, 0, grow=False)
    ip, ids = qf.indptr, np.minimum(qf.ids, V)
    order = sorted(range(q), key=lambda i: ids[ip[i]:ip[i + 1]].tolist())     # text order, ties by index (stable)
    distinct, per_query = [], []
    cover = {kt: [] for kt in (0, 64, 96, 128, 192, 256)}
    warp_iters = {kt: [] for kt in cover}  # per 32-query warp: the most F2 features one of its queries has left over
    for t0 in range(0, q - TILE + 1, TILE):
        counts = {}
        tot = 0
        tile_feats = []
        for i in order[t0:t0 + TILE]:
            feats = [f for f in ids[ip[i]:ip[i + 1]].tolist() if f2[f]]
            tile_feats.append(feats)
            per_query.append(len(feats))
            tot += len(feats)
            for f in feats:
                counts[f] = counts.get(f, 0) + 1
        distinct.append(len(counts))
        ranked = sorted(counts, key=lambda f: (-counts[f], f))  # the dictionary's order: count descending, lower id first
        for kt in cover:
            d = set(ranked[:kt])
            left = [sum(1 for f in feats if f not in d) for feats in tile_feats]
            cover[kt].append(1 - sum(left) / max(tot, 1))
            for w in range(0, TILE, 32):
                warp_iters[kt].append(max(left[w:w + 32]))
    d = np.array(distinct)
    pq = np.array(per_query)
    print(f"queries {q}: F2 features per query: mean {pq.mean():.1f}, p99 {np.percentile(pq, 99):.0f}, > Q2CAP={Q2CAP}: {(pq > Q2CAP).mean() * 100:.2f} %")
    print(f"distinct F2 features per {TILE}-query tile: mean {d.mean():.0f}, median {np.median(d):.0f}, p90 {np.percentile(d, 90):.0f}, max {d.max()}")
    for kt, c in cover.items():
        c, wi = np.array(c), np.array(warp_iters[kt])
        print(f"  dictionary of {kt:3d} columns covers {c.mean() * 100:5.1f} % of the tile's (query, F2 feature) incidences "
              f"(p10 {np.percentile(c, 10) * 100:5.1f} %); per-warp loop over the rest: mean {wi.mean():.2f}, max {wi.max()} iterations")
    qf.close()


if __name__ == "__main__":
    main()
