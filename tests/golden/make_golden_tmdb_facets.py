"""TMDB facet codes fixture: two per-document category columns of the TMDB corpus, in the doc order of
tests/golden/tmdb_index.npz (the fixture's key order, as make_golden_tmdb.load_corpus reads it), for the facet
counts of the batched top-k on machines without the reference tree.

    python tests/golden/make_golden_tmdb_facets.py      (build container only)

Writes tests/golden/tmdb_facets.npz:
  original_language        int32[n_docs]: index into original_language.names (the sorted language codes), -1 for
                           a film whose language is missing or empty
  original_language.names  the language codes, "\\n"-joined as bytes
  decade                   int32[n_docs]: (release year // 10) - first decade // 10, -1 for a film without a date
  decade.first             the first decade (a year)
"""
import gzip
import json
import os

import numpy as np

from make_golden import HERE
from make_golden_tmdb import FIXTURE


def main():
    with gzip.open(FIXTURE) as f:
        raw = json.load(f)
    langs = [raw[doc_id].get("original_language") or "" for doc_id in raw.keys()]
    dates = [raw[doc_id].get("release_date") or "" for doc_id in raw.keys()]
    names = sorted(set(x for x in langs if x))
    lang = np.asarray([names.index(x) if x else -1 for x in langs], dtype=np.int32)
    years = np.asarray([int(d[:4]) if d else -1 for d in dates], dtype=np.int64)
    first = int(years[years >= 0].min()) // 10 * 10
    decade = np.where(years >= 0, years // 10 - first // 10, -1).astype(np.int32)
    out = os.path.join(HERE, "tmdb_facets.npz")
    np.savez_compressed(out, **{"original_language": lang,
                                "original_language.names": np.frombuffer("\n".join(names).encode(), dtype=np.uint8),
                                "decade": decade, "decade.first": np.asarray(first)})
    print(out, len(lang), "docs,", len(names), "languages,", int(decade.max()) + 1, "decades,",
          int((lang < 0).sum()), "without a language,", int((decade < 0).sum()), "without a date")


if __name__ == "__main__":
    main()
