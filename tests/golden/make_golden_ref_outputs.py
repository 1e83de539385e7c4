"""Stores what the REAL reference computes on inputs too large to commit whole, so that the tests which
compare against it run from the repository alone:

  * op_pairs.npz -- contiguous slices of the reference's seven saved posting pairs
    (fixtures/{lhs,rhs,mask}_*.npy, test_snp_ops.py:324-350), each centred on a match, with the
    reference's intersect / intersect_with_adjacents output on exactly those slices
    (tests/test_op_tables.py::test_saved_posting_pairs);
  * ref_synth.json -- SHA-256 digests of the reference's docfreq / termfreqs / score vectors on the seeded
    300k-doc synthetic corpus (tests/test_ref_cpu.py).

    python tests/golden/make_golden_ref_outputs.py <reference source tree>

The reference is imported from oracle/_ref, which oracle/build_ref.py builds from the given tree with
`pip install --no-index --no-build-isolation --no-deps --target oracle/_ref` (its setup.py cythonizes the
roaringish ops; Cython must be installed).  The script refuses to run unless those ops are the compiled extension
modules under oracle/_ref, and it first reproduces the reference's full-pair digests recorded in op_tables.json
by make_golden_op_tables.py.  Both files record the reference's version and the extension modules that produced
them under "reference".  Only inputs and outputs are written; everything is seeded, so re-running reproduces the
files.
"""
import hashlib
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

SUFFIXES = (128, 185, 24179, 27685, 44358, 45907, 90596)
LHS_HALF, RHS_HALF = 256, 512


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def reference_provenance():
    """The reference package in oracle/_ref and its compiled native ops (raises if they are not extension modules)."""
    import importlib.metadata
    from oracle.build_ref import REF_DST, import_reference
    import_reference()
    import searcharray.roaringish  # noqa: F401
    from searcharray.roaringish.intersect import intersect_with_adjacents  # noqa: F401
    native = sorted(m for m in sys.modules if m.startswith("searcharray.roaringish.")
                    and getattr(sys.modules[m], "__file__", "").endswith(".so"))
    for m in ("searcharray.roaringish.intersect", "searcharray.roaringish.popcount"):
        f = sys.modules[m].__file__
        assert f.endswith(".so") and os.path.realpath(f).startswith(os.path.realpath(REF_DST)), f
    dist = [f"{d.metadata['Name']} {d.version}" for d in importlib.metadata.distributions(path=[REF_DST])]
    return {"package": dist, "native_ops": [os.path.basename(sys.modules[m].__file__) for m in native],
            "built_by": "oracle/build_ref.py: pip install --no-index --no-build-isolation --no-deps --target oracle/_ref"}


def digest(a):
    return hashlib.sha256(np.ascontiguousarray(a, dtype=np.uint64).tobytes()).hexdigest()


def op_pairs(fixtures, provenance):
    from searcharray.roaringish import intersect
    from searcharray.roaringish.intersect import intersect_with_adjacents
    with open(os.path.join(HERE, "op_tables.json")) as f:
        recorded = {r["suffix"]: r for r in json.load(f)["fixtures"]}
    out = {"reference": np.asarray(json.dumps(provenance))}
    for suffix in SUFFIXES:
        lhs = np.load(os.path.join(fixtures, f"lhs_{suffix}.npy"))
        rhs = np.load(os.path.join(fixtures, f"rhs_{suffix}.npy"))
        mask = np.load(os.path.join(fixtures, f"mask_{suffix}.npy"))
        li, ri = intersect(lhs, rhs, mask=mask)
        # the whole pair first: the same answers the reference gave when op_tables.json was made
        rec = recorded[suffix]
        assert (len(lhs), len(rhs), int(mask)) == (rec["n_lhs"], rec["n_rhs"], rec["mask"]), suffix
        assert [len(li), digest(li), digest(ri)] == rec["intersect"], suffix
        full_adj = intersect_with_adjacents(lhs, rhs, mask=mask)
        assert [[len(x), digest(x)] for x in full_adj] == rec["with_adjacents"], suffix
        cl, cr = (int(li[len(li) // 2]), int(ri[len(ri) // 2])) if len(li) else (len(lhs) // 2, len(rhs) // 2)
        ls = np.ascontiguousarray(lhs[max(0, cl - LHS_HALF):cl + LHS_HALF])
        rs = np.ascontiguousarray(rhs[max(0, cr - RHS_HALF):cr + RHS_HALF])
        sli, sri = intersect(ls, rs, mask=mask)
        adj = intersect_with_adjacents(ls, rs, mask=mask)
        out.update({f"{suffix}.lhs": ls, f"{suffix}.rhs": rs, f"{suffix}.mask": np.asarray(mask, dtype=np.uint64),
                    f"{suffix}.lhs_idx": sli, f"{suffix}.rhs_idx": sri})
        for i, a in enumerate(adj):
            out[f"{suffix}.adj{i}"] = a
        print(suffix, len(ls), len(rs), len(sli), [len(a) for a in adj])
    path = os.path.join(HERE, "op_pairs.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path))


def ref_synth(provenance):
    from oracle import ref_runner
    from searcharray_b200 import synth
    spec = synth.SynthSpec(300_000, terms_per_bucket=5, n_phrases=16, n_bigrams=4)
    host, _, _ = synth.generate_shard(spec)
    avgdl = synth.global_avg_doc_length(spec)
    arr = ref_runner.reference_array(host, avg_doc_length=avgdl)
    sim = ref_runner.bm25(1.2, 0.75)
    out = {"reference": provenance, "terms": {}, "phrases": [], "slop2": []}
    for name, _, _ in spec.terms:
        out["terms"][name] = {"df": int(arr.docfreq(name)), "tf": sha(arr.termfreqs(name)),
                              "score": sha(arr.score(name, similarity=sim))}
    out["missing_score"] = sha(arr.score("nope"))
    for ph in spec.phrases:
        tf = arr.termfreqs(ph["terms"])
        out["phrases"].append({"terms": ph["terms"], "tf": sha(tf), "nonzero": int(np.count_nonzero(tf)),
                               "score": sha(arr.score(ph["terms"], similarity=sim))})
    for ph in spec.phrases[::3]:
        out["slop2"].append({"terms": ph["terms"], "tf": sha(arr.termfreqs(ph["terms"], slop=2))})
    path = os.path.join(HERE, "ref_synth.json")
    with open(path, "w") as f:
        json.dump(out, f, indent=0)
    print(path, os.path.getsize(path))


if __name__ == "__main__":
    prov = reference_provenance()
    op_pairs(os.path.join(sys.argv[1], "fixtures"), prov)
    ref_synth(prov)
