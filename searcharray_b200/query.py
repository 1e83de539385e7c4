"""Boolean queries for SearchArray.search_topk: OR / AND / min-should-match over term and phrase clauses, and
Lucene-style required / optional / filter / prohibited clauses with per-clause boosts.

Or(clauses, mm) ranks, per doc, s = score(c0) + score(c1) + ... (float32, folded left in clause order) among the docs
where at least mm clauses score > 0 -- the reference's own composition of multi-clause queries
(test/test_search.py:126-226) -- and search_topk returns the top k of it by (score desc, doc asc), computed on the
device (sa_score_batch_topk_bool).  Bool(must, should, filter, must_not, mm) and Boost(clause, weight) extend that
composition.  Field(field, clause) names the DataFrame column a clause scores on, for queries over several columns
(solr.fields_topk, sa_multi_score_batch_topk_bool).  DisMax(clauses, tie) is one clause scored by its best member
plus tie times the others (Lucene's DisjunctionMaxQuery).  An Or / And / Bool may itself be a clause of another (a
nested query, scored by what it ranks as a query of its own).  Feature(name, function) is a leaf scored by a
per-document numeric column registered with SearchArray.set_feature (Lucene's FeatureField).  Range(name, ...) and
In(name, codes) are filter leaves over a feature column and a facet column (SearchArray.set_facet), scored 1 where
they match (Elasticsearch's range and terms queries).  The device entry points take the queries flattened for their
form (bool_form, flatten_bool)."""
import math
import numbers
from typing import List, NamedTuple, Optional, Union

import numpy as np

from .solr import parse_min_should_match

SA_BOOL_MAX_CLAUSES = 64          # include/searcharray_b200.h
SA_BOOL_MAX_NESTED = 64           # nested queries in one top-level query, at any depth
SA_NO_NODE = 0xFFFFFFFF           # include/searcharray_b200.h
ED_MAX_FIELDS = 8                 # fields of one sa_multi (sa_multi.cuh)
SA_MAX_PHRASE_TERMS = 16          # include/searcharray_b200.h
ED_MAX_ROWS = 64                  # phrase rows of one field in one sa_multi_phrases call (sa_multi.cuh)
ED_MAX_PHASE_ENTRIES = ED_MAX_FIELDS * SA_MAX_PHRASE_TERMS   # entries of one sa_multi_add_phase call (sa_multi.cuh)
SA_OCCUR_SHOULD, SA_OCCUR_MUST, SA_OCCUR_FILTER, SA_OCCUR_MUST_NOT = 0, 1, 2, 3
SA_MAX_FEATURES = 16              # include/searcharray_b200.h
SA_FEATURE_TERM_BASE = 0xFF000000
SA_MAX_FACETS = 8                 # include/searcharray_b200.h: facet columns of one index
SA_FACET_MAX_BUCKETS = 1024       # include/searcharray_b200.h
SA_BOOL_MAX_FACETS = 4            # include/searcharray_b200.h: facets counted in one call
SA_MAX_GROUPS = 4                 # include/searcharray_b200.h: group columns of one index
FEATURE_FUNCTIONS = {"linear": 0, "saturation": 1, "log": 2}     # SA_FEATURE_LINEAR, _SATURATION, _LOG
SA_FEATURE_RANGE, SA_FEATURE_IN = 0x10, 0x11                       # include/searcharray_b200.h

Clause = Union[str, List[str]]


def _clause(c):
    """A clause as search_topk's query form: str (term) or list[str] (phrase), a Feature, Range or In, a Field of one,
    a DisMax, or a nested Or / And / Bool; anything else is a TypeError."""
    if isinstance(c, (str, Feature, Range, In, Field, DisMax, Or, Bool)):
        return c
    if isinstance(c, (list, tuple)) and c and all(isinstance(t, str) for t in c):
        return list(c)
    raise TypeError(f"a clause is a str (term) or a non-empty list of str (phrase), not {c!r}")


class Feature:
    """A clause scored by a per-document numeric column of the array's index (SearchArray.set_feature): Lucene's
    FeatureField, Elasticsearch's rank_feature -- popularity, votes, a quality score added to the text score.  With x
    the doc's value, v = 0 where x is 0, and otherwise:

      "linear"      v = x
      "saturation"  v = x / (x + pivot), in float32 (pivot finite and > 0)
      "log"         v = float32(log(float64(scaling_factor) + float64(x))) (scaling_factor finite and >= 1)

    Parameters are rounded to float32 once; a missing, extra or out-of-range one is a ValueError, a name that is not a
    str a TypeError.  A Feature is a leaf like a term: it matches where v > 0, counts once towards mm, adds w * v under
    must / should (Boost(Feature(...), w)) and plays a leaf's role under filter / must_not.  It is accepted in Or,
    And, every list of Bool and nested queries; in solr.fields_topk as Field(column, Feature(...)), the column whose
    index holds the values.  Range and In, the filter leaves over the same columns and over facet columns, are
    accepted and refused exactly where a Feature is.  It is not a DisMax member (TypeError), and not a query of its own in search_topk
    (TypeError: write Bool(should=[Feature(...)])).  apply(x) is the transform in numpy."""

    def __init__(self, name, function="linear", pivot=None, scaling_factor=None):
        if not isinstance(name, str):
            raise TypeError(f"a feature name is a str, not {name!r}")
        if function not in FEATURE_FUNCTIONS:
            raise ValueError(f"a feature function is one of {sorted(FEATURE_FUNCTIONS)}, not {function!r}")
        need = {"linear": None, "saturation": "pivot", "log": "scaling_factor"}[function]
        for key, value in (("pivot", pivot), ("scaling_factor", scaling_factor)):
            if key == need and value is None:
                raise ValueError(f"a {function} feature needs {key}")
            if key != need and value is not None:
                raise ValueError(f"a {function} feature takes no {key}")
        param = np.float32(0.0)
        if need is not None:
            value = pivot if need == "pivot" else scaling_factor
            with np.errstate(over="ignore"):
                param = np.float32(float(value))
            low_ok = param > 0 if need == "pivot" else param >= 1
            if not (np.isfinite(param) and low_ok):
                raise ValueError(f"a {function} feature's {need} is finite and {'> 0' if need == 'pivot' else '>= 1'}"
                                 f" in float32, not {value!r}")
        self.name, self.function, self.param = name, function, param

    @property
    def fn(self):
        """The SA_FEATURE_* code of the function."""
        return FEATURE_FUNCTIONS[self.function]

    def term_id(self, slot):
        """The reserved term id (SA_FEATURE_TERM) naming this function on feature slot `slot` of an index."""
        return SA_FEATURE_TERM_BASE | (self.fn << 8) | int(slot)

    def apply(self, x):
        """v = f(x) as float32[len(x)], as the device computes it: 0 where x is not > 0."""
        x = np.asarray(x, dtype=np.float32)
        pos = x > 0
        if self.function == "linear":
            v = x
        elif self.function == "saturation":
            with np.errstate(under="ignore"):
                v = x / (x + self.param)
        else:
            v = np.log(np.float64(self.param) + x.astype(np.float64)).astype(np.float32)
        return np.where(pos, v, np.float32(0)).astype(np.float32)

    def __repr__(self):
        extra = {"linear": "", "saturation": f", pivot={float(self.param)!r}",
                 "log": f", scaling_factor={float(self.param)!r}"}[self.function]
        return f"Feature({self.name!r}, {self.function!r}{extra})"


def _bits(x):
    """The bit pattern of float32 x as an int (the C ABI's encoding of a range bound)."""
    return int(np.float32(x).view(np.uint32))


def _f32_bound(a, up, strict):
    """The float32 nearest a in one direction, as a float: up, the least float32 >= a (> a if strict); down, the
    greatest float32 <= a (< a if strict).  +-inf beyond float32's range, so that x >= result is exactly x >= a
    (x > a, x <= a, x < a) for every finite float32 x."""
    big = float(np.finfo(np.float32).max)
    if a > big:
        return math.inf
    if a < -big:
        return -math.inf
    f = np.float32(a)
    with np.errstate(over="ignore"):        # past the largest float32: inf, as wanted
        f = _f32_step(f, a, up, strict)
    return float(f)


def _f32_step(f, a, up, strict):
    """f, the float32 nearest a, stepped one float32 outward where it lies on the wrong side of a."""
    if up and (float(f) < a or (strict and float(f) == a)):
        f = np.nextafter(f, np.float32(np.inf))
    if not up and (float(f) > a or (strict and float(f) == a)):
        f = np.nextafter(f, np.float32(-np.inf))
    return f


class Range:
    """A filter leaf over a feature column (SearchArray.set_feature): Elasticsearch's range query, Lucene's point range.
    It matches the docs whose value x in column `name` is inside the bounds given -- gt (x > gt), gte (x >= gte), lt
    (x < lt), lte (x <= lte) -- and never a doc whose value is 0 (the column's "no value", as Elasticsearch skips docs
    without the field).  The comparison is exact between x (a float32, widened to float64) and each bound as given:
    the device compares x with float32 bounds rounded outward (bounds()), which selects the same docs.  Columns hold
    float32, so a value above 2^24 (epoch seconds, say) was rounded when it was set.

    At least one bound; gt with gte, or lt with lte, a NaN or infinite bound is a ValueError; a bound that is a bool or
    not a real number a TypeError.  An empty range (gte=5, lt=5) is accepted and matches nothing.  It scores as a
    constant: 1 where it matches, 0 elsewhere, and is otherwise a leaf like a Feature -- it counts once towards mm, adds
    w * 1 under must / should (Boost(Range(...), w)), and plays a leaf's role under filter / must_not.  It is accepted
    and refused where a Feature is (not a DisMax member, not a query of its own: write Bool(filter=[...])); in
    solr.fields_topk as Field(column, Range(...)).  match(x) is the filter in numpy."""

    def __init__(self, name, gt=None, gte=None, lt=None, lte=None):
        if not isinstance(name, str):
            raise TypeError(f"a range's column name is a str, not {name!r}")
        given = {}
        for key, v in (("gt", gt), ("gte", gte), ("lt", lt), ("lte", lte)):
            if v is None:
                continue
            if isinstance(v, (bool, np.bool_)) or not isinstance(v, numbers.Real):
                raise TypeError(f"a range bound is a real number, not {key}={v!r}")
            try:
                x = float(v)
            except OverflowError:           # an int beyond float64: beyond every float32 too
                x = math.inf if v > 0 else -math.inf
            else:
                if not math.isfinite(x):
                    raise ValueError(f"a range bound is finite, not {key}={v!r}")
            given[key] = x
        if not given:
            raise ValueError("a range needs at least one bound (gt, gte, lt or lte)")
        if "gt" in given and "gte" in given:
            raise ValueError("a range takes gt or gte, not both")
        if "lt" in given and "lte" in given:
            raise ValueError("a range takes lt or lte, not both")
        self.name = name
        self.gt, self.gte, self.lt, self.lte = (given.get(k) for k in ("gt", "gte", "lt", "lte"))

    def bounds(self):
        """(lo, hi): the float32 interval [lo, hi] (as floats) the device tests x against, the bounds rounded
        outward; -inf / +inf where a side is open or a bound lies beyond float32's range."""
        lo, hi = -math.inf, math.inf
        if self.gte is not None:
            lo = _f32_bound(self.gte, True, False)
        if self.gt is not None:
            lo = _f32_bound(self.gt, True, True)
        if self.lte is not None:
            hi = _f32_bound(self.lte, False, False)
        if self.lt is not None:
            hi = _f32_bound(self.lt, False, True)
        return lo, hi

    def entries(self, slot):
        """The clause entries of the C ABI on feature slot `slot`: SA_RANGE_TERM(slot), then lo's and hi's bits."""
        lo, hi = self.bounds()
        return [SA_FEATURE_TERM_BASE | (SA_FEATURE_RANGE << 8) | int(slot), _bits(lo), _bits(hi)]

    def match(self, x):
        """bool[len(x)]: where the float32 values x (widened to float64) are > 0 and inside the bounds."""
        x = np.asarray(x, dtype=np.float32).astype(np.float64)
        m = x > 0
        if self.gt is not None:
            m &= x > self.gt
        if self.gte is not None:
            m &= x >= self.gte
        if self.lt is not None:
            m &= x < self.lt
        if self.lte is not None:
            m &= x <= self.lte
        return m

    def __repr__(self):
        shown = "".join(f", {k}={v!r}" for k, v in (("gt", self.gt), ("gte", self.gte), ("lt", self.lt),
                                                    ("lte", self.lte)) if v is not None)
        return f"Range({self.name!r}{shown})"


class In:
    """A filter leaf over a facet column (SearchArray.set_facet): Elasticsearch's terms query on a keyword field,
    Lucene's TermInSetQuery.  It matches the docs whose code in column `name` is one of `codes`, never a doc without a
    value (code -1).  codes: a non-empty list (tuple, or integer array) of ints >= 0, duplicates allowed; each must be
    below the facet's n_buckets, which is checked when the call is prepared (ValueError, before any device work).  A
    non-list or a non-int code is a TypeError, an empty list or a negative code a ValueError.  It scores and is
    accepted and refused as Range.  match(codes) is the filter in numpy."""

    def __init__(self, name, codes):
        if not isinstance(name, str):
            raise TypeError(f"a facet name is a str, not {name!r}")
        if isinstance(codes, np.ndarray):
            if codes.dtype.kind not in "iu":
                raise TypeError(f"In codes are ints, not dtype {codes.dtype}")
            codes = codes.tolist()
        if not isinstance(codes, (list, tuple)):
            raise TypeError(f"In codes are a list of ints, not {codes!r}")
        out = []
        for c in codes:
            if isinstance(c, (bool, np.bool_)) or not isinstance(c, (int, np.integer)):
                raise TypeError(f"an In code is an int, not {c!r}")
            out.append(int(c))
        if not out:
            raise ValueError("an In clause needs at least one code")
        if min(out) < 0:
            raise ValueError(f"In codes are >= 0: {out}")
        self.name, self.codes = name, out

    def entries(self, slot):
        """The clause entries of the C ABI on facet slot `slot`: SA_IN_TERM(slot), then the codes."""
        return [SA_FEATURE_TERM_BASE | (SA_FEATURE_IN << 8) | int(slot)] + self.codes

    def match(self, codes):
        """bool[len(codes)]: where the codes (-1: no value) are in the set."""
        codes = np.asarray(codes)
        return (codes >= 0) & np.isin(codes, self.codes)

    def __repr__(self):
        return f"In({self.name!r}, {self.codes!r})"


COLUMN_CLAUSES = (Feature, Range, In)     # leaves scored from a column of the index, not from its postings


def _is_feature(c):
    """Whether a clause (without its Boost) is a Feature, Range or In, or a Field of one."""
    return isinstance(c, COLUMN_CLAUSES) or (isinstance(c, Field) and isinstance(c.clause, COLUMN_CLAUSES))


class Field:
    """A term (str) or phrase (non-empty list of str) clause scored on the DataFrame column `field`, as
    frame[field].array.score(clause) scores it -- Lucene's `title:star`.  Accepted wherever a clause is (Or, And, the
    four lists of Bool) by solr.fields_topk, which needs every clause to name its field; SearchArray.search_topk
    refuses it.  A boosted field clause is Boost(Field(field, clause), weight); a Field holds no Boost or Field.
    Field(field, Feature(...)) is a feature clause whose values are those set on that column's index, and
    Field(field, Range(...)) / Field(field, In(...)) filter on that index's feature / facet columns."""

    def __init__(self, field, clause):
        if not isinstance(field, str):
            raise TypeError(f"a field is a column name (str), not {field!r}")
        if isinstance(clause, (Boost, Field, DisMax, Or, Bool)):
            raise TypeError(f"a Field holds a term or a phrase; boost a field clause as Boost(Field(...), w), not {clause!r}")
        self.field = field
        self.clause = _clause(clause)

    def __repr__(self):
        return f"Field({self.field!r}, {self.clause!r})"


class Boost:
    """A term or phrase clause whose score is multiplied by `weight` (Lucene's `title^2`) before it is added:
    s = s + float32(weight) * score(clause), the product rounded to float32.  `weight` is finite and >= 0 and is
    rounded to float32 once.  A doc still counts as matched by the clause where its unweighted score is > 0, so a
    weight of 0 matches without scoring.  Accepted where a clause scores: in Or, And, Bool's must and should.  A
    nested Or / And / Bool may be boosted the same way: it adds float32(weight) * (what it ranks)."""

    def __init__(self, clause, weight):
        if isinstance(clause, DisMax):
            raise TypeError(f"a DisMax takes no Boost: boost its members instead, as edismax's qf boosts do: {clause!r}")
        self.clause = _clause(clause)
        w = float(weight)
        if not math.isfinite(w) or w < 0:
            raise ValueError(f"a boost is finite and >= 0, not {weight!r}")
        self.weight = np.float32(w)

    def __repr__(self):
        return f"Boost({self.clause!r}, {float(self.weight)!r})"


def _scoring(clauses):
    """(clauses, float32 weights) of a list of clauses and Boosts."""
    out, weights = [], []
    for c in clauses:
        if isinstance(c, Boost):
            out.append(c.clause)
            weights.append(c.weight)
        else:
            out.append(_clause(c))
            weights.append(np.float32(1.0))
    return out, weights


class DisMax:
    """One clause scored by its best member: Lucene's DisjunctionMaxQuery, Elasticsearch's dis_max, the per-term qf
    part of edismax.  With v_j = float32(w_j * score(c_j)) (w_j the member's Boost, 1 without one),
    d = m + (t - m) * tie, m = max_j v_j, t = v_0 + v_1 + ... folded left in member order, every operation rounded to
    float32.  The DisMax matches a doc where any member scores > 0 (unweighted, so a zero-weight member still matches).

    clauses: at least one member, each a term (str), a phrase (list[str], matched with the call's slop), a Field of
    either, or a Boost of any of these; a DisMax, Or, And or Bool member is a TypeError.  tie: finite, in [0, 1],
    rounded to float32 once.  Accepted wherever a clause is (Or, And, the four lists of Bool), where it is one clause
    (it counts once towards mm and adds d with weight 1); as a query of its own it is Bool(should=[it]).  It takes no
    Boost itself.  Members need sparse-safe BM25 parameters (k1 > 0, 0 <= b < 1), as phrase clauses do.
    DisMax([c]) scores exactly as c."""

    def __init__(self, clauses, tie=0.0):
        clauses = list(clauses)
        if not clauses:
            raise ValueError("a DisMax needs at least one member")
        for c in clauses:
            inner = c.clause if isinstance(c, Boost) else c
            if isinstance(inner, (DisMax, Or, Bool)) or _is_feature(inner):
                raise TypeError(f"a DisMax member is a term, a phrase or a Field of one (boosted or not), not {c!r}")
        self.clauses, self.weights = _scoring(clauses)
        t = float(tie)
        if not math.isfinite(t) or not 0.0 <= t <= 1.0:
            raise ValueError(f"a DisMax tie is finite and in [0, 1], not {tie!r}")
        self.tie = np.float32(t)
        _check_count(len(self.clauses))

    @property
    def boosted(self):
        """Whether any member has a weight other than 1."""
        return any(w != 1.0 for w in self.weights)

    def __repr__(self):
        shown = [Boost(c, w) if w != 1.0 else c for c, w in zip(self.clauses, self.weights)]
        return f"DisMax({shown!r}, tie={float(self.tie)!r})"


def _inner(c):
    """A clause without its Boost."""
    return c.clause if isinstance(c, Boost) else c


def _is_node(c):
    """Whether a clause (boosted or not) is a nested Or / And / Bool."""
    return isinstance(_inner(c), (Or, Bool))


def _n_clauses(clauses):
    """The leaves a list holds as the device counts them: a DisMax counts its members, a nested query its leaves."""
    return sum(_inner(c).n_leaves if _is_node(c) else len(c.clauses) if isinstance(c, DisMax) else 1 for c in clauses)


def _n_nodes(clauses):
    """The nested queries a list holds, at any depth; a query object used twice counts twice."""
    return sum(1 + _inner(c).n_nested for c in clauses if _is_node(c))


def _check_count(n):
    if n > SA_BOOL_MAX_CLAUSES:
        raise ValueError(f"a boolean query has at most {SA_BOOL_MAX_CLAUSES} clauses, not {n}")


def _check_nodes(n):
    if n > SA_BOOL_MAX_NESTED:
        raise ValueError(f"a boolean query holds at most {SA_BOOL_MAX_NESTED} nested queries, not {n}")


class Or:
    """A query matching docs where at least `mm` of `clauses` score > 0, scored by the sum of the clauses' scores.

    clauses: a str (a term), a list[str] (a phrase, matched with search_topk's `slop`) or a Boost of either;
    duplicates count twice.  mm: an int or a Solr min-should-match spec ("2", "-1", "75%", "2<-25%"), clamped to
    [0, len(clauses)] as edismax clamps it (solr.parse_min_should_match).

    A clause may also be a nested Or / And / Bool N (or a Boost of one), at any depth.  It is one clause: its score
    at doc d is r_N(d), what N ranks d with as a query of its own (its sum where all its conditions hold and the sum
    is > 0, else 0), it matches where r_N(d) > 0 and counts once towards mm.  So, unlike Lucene, a nested query whose
    sum is <= 0 (all its boosts 0, say) does not match.  Or([a, Or([b])]) scores as Or([a, b]); flattening a larger
    nested Or in general changes the fold order and the mm counts.  A top-level query holds at most
    SA_BOOL_MAX_CLAUSES leaves in its whole tree (DisMax members counted) and SA_BOOL_MAX_NESTED nested queries; a
    sub-query object used twice counts twice."""

    def __init__(self, clauses, mm=1):
        clauses = list(clauses)
        if not clauses:
            raise ValueError("a boolean query needs at least one clause")
        self.n_leaves, self.n_nested = _n_clauses(clauses), _n_nodes(clauses)
        _check_count(self.n_leaves)
        _check_nodes(self.n_nested)
        self.clauses, self.weights = _scoring(clauses)
        self.mm = parse_min_should_match(len(self.clauses), str(mm))
        self.form = _form(self.clauses, self.boosted)       # bool_form

    @property
    def boosted(self):
        """Whether any clause has a weight other than 1 (such a query takes the OCCUR form)."""
        return any(w != 1.0 for w in self.weights)

    def __repr__(self):
        if self.boosted:
            shown = [Boost(c, w) if w != 1.0 else c for c, w in zip(self.clauses, self.weights)]
            return f"{type(self).__name__}({shown!r}, mm={self.mm})"
        return f"{type(self).__name__}({self.clauses!r}, mm={self.mm})"


class And(Or):
    """Every clause must score > 0: Or(clauses, mm=len(clauses))."""

    def __init__(self, clauses):
        clauses = list(clauses)
        super().__init__(clauses, mm=len(clauses))


class Bool:
    """Lucene's boolean query: a doc ranks iff every `must` and `filter` clause scores > 0 there, no `must_not`
    clause does, at least `mm` of the `should` clauses do, and s > 0, where
    s = w0 * score(c0) + w1 * score(c1) + ... over must + should in that order (float32, each product rounded, folded
    left).  `filter` and `must_not` clauses add nothing to s and take no Boost.

    mm counts `should` clauses only: an int or a Solr spec (solr.parse_min_should_match(len(should), str(mm))); by
    default 0 when there are must or filter clauses, else 1.  At least one must or should clause is needed (without
    one nothing can score > 0), and at most SA_BOOL_MAX_CLAUSES clauses in the four lists together.  Every list
    accepts a nested Or / And / Bool as Or does (a Boost of one in must and should only); under filter / must_not it
    plays a leaf's role, matching where what it ranks is > 0."""

    def __init__(self, must=(), should=(), filter=(), must_not=(), mm=None):
        must, should, filter, must_not = list(must), list(should), list(filter), list(must_not)
        for role, cs in (("filter", filter), ("must_not", must_not)):
            for c in cs:
                if isinstance(c, Boost) or (isinstance(c, DisMax) and c.boosted):
                    raise ValueError(f"a {role} clause adds nothing to the score and takes no Boost: {c!r}")
        self.must, self.must_weights = _scoring(must)
        self.should, self.should_weights = _scoring(should)
        self.filter = [_clause(c) for c in filter]
        self.must_not = [_clause(c) for c in must_not]
        if not self.must and not self.should:
            raise ValueError("a Bool query needs at least one must or should clause: nothing else scores")
        every = must + should + filter + must_not
        self.n_leaves, self.n_nested = _n_clauses(every), _n_nodes(every)
        _check_count(self.n_leaves)
        _check_nodes(self.n_nested)
        if mm is None:
            mm = 0 if (self.must or self.filter) else 1
        self.mm = parse_min_should_match(len(self.should), str(mm))
        self.form = _form(self.must + self.should + self.filter + self.must_not, True)   # bool_form

    def occur_clauses(self):
        """(clauses, float32 weights, occurs) in the order the device folds them: must, should, filter, must_not."""
        clauses = self.must + self.should + self.filter + self.must_not
        one = np.float32(1.0)
        weights = self.must_weights + self.should_weights + [one] * (len(self.filter) + len(self.must_not))
        occurs = ([SA_OCCUR_MUST] * len(self.must) + [SA_OCCUR_SHOULD] * len(self.should) +
                  [SA_OCCUR_FILTER] * len(self.filter) + [SA_OCCUR_MUST_NOT] * len(self.must_not))
        return clauses, weights, occurs

    def __repr__(self):
        def shown(cs, ws):
            return [Boost(c, w) if w != 1.0 else c for c, w in zip(cs, ws)]
        return (f"Bool(must={shown(self.must, self.must_weights)!r}, "
                f"should={shown(self.should, self.should_weights)!r}, filter={self.filter!r}, "
                f"must_not={self.must_not!r}, mm={self.mm})")


def is_boolean(q):
    """Whether search_topk routes q to the boolean path."""
    return isinstance(q, (Or, Bool, DisMax))


def _top_clauses(q):
    """The clauses of an Or / And / Bool, or a top-level DisMax as the one clause it is."""
    if isinstance(q, DisMax):
        return [q]
    return q.occur_clauses()[0] if isinstance(q, Bool) else q.clauses


def _leaves(q):
    """Every clause of a boolean query's tree that is not a nested query: its DisMax clauses and their members, and
    the leaves of its nested queries at any depth."""
    for c in _top_clauses(q):
        if isinstance(c, (Or, Bool)):
            yield from _leaves(c)
        else:
            yield c
            if isinstance(c, DisMax):
                yield from c.clauses


def has_field(q):
    """Whether a boolean query holds a Field clause (solr.fields_topk's form), a DisMax's members and nested queries
    included."""
    return any(isinstance(c, Field) for c in _leaves(q))


def has_dismax(q):
    """Whether q is or holds a DisMax (the DISMAX form), nested queries included."""
    return any(isinstance(c, DisMax) for c in _leaves(q))


def has_feature(q):
    """Whether a boolean query holds a column clause (Feature, Range or In, or a Field of one), nested queries
    included: such a query runs at least at the OCCUR form."""
    return any(_is_feature(c) for c in _leaves(q))


def is_nested(q):
    """Whether a boolean query holds a nested Or / And / Bool (the NESTED form)."""
    return not isinstance(q, DisMax) and any(isinstance(c, (Or, Bool)) for c in _top_clauses(q))


def needs_occur(q):
    """Whether q takes at least the OCCUR form: a Bool, an Or / And with a weight other than 1 or a feature clause."""
    return isinstance(q, Bool) or q.boosted or has_feature(q)


# The forms of a boolean batch, ordered: each form's arrays are those of the one before plus its own, and the C entry
# points run the instance the non-NULL arrays select.
OR_AND, OCCUR, DISMAX, NESTED = 1, 2, 3, 4


def bool_form(q):
    """The form a boolean query takes: NESTED if it holds a nested Or / And / Bool, else DISMAX if it is or holds a
    DisMax, else OCCUR if it is a Bool, has a weight other than 1 or a feature clause, else OR_AND."""
    return DISMAX if isinstance(q, DisMax) else q.form


def _form(clauses, occur):
    """bool_form of an Or / And / Bool with these top-level clauses (Boosts removed); occur: it is a Bool or boosted.
    Without a nested query, every DisMax of the tree is a top-level clause."""
    form = OCCUR if occur else OR_AND
    for c in clauses:
        if isinstance(c, (Or, Bool)):
            return NESTED
        if isinstance(c, DisMax):
            form = DISMAX
        elif _is_feature(c):       # the FEATURE instances start at the roles form
            form = max(form, OCCUR)
    return form


class BoolBatch(NamedTuple):
    """Boolean queries as sa_score_batch_topk_bool takes them (flatten_bool).  Arrays the form does not use are None,
    passed as NULL."""
    clauses: list                   # per clause: search_topk's query form (str, list[str], Feature, Range or In);
                                    # None for a nested clause
    node_starts: np.ndarray         # uint32: node n's clauses are [node_starts[n], node_starts[n + 1])
    clause_node: Optional[np.ndarray]   # uint32 per clause: its nested node, else SA_NO_NODE (NESTED)
    mm: np.ndarray                  # uint32 per node
    weights: Optional[np.ndarray]   # float32 per clause (OCCUR up)
    occurs: Optional[np.ndarray]    # uint8 SA_OCCUR_* per clause (OCCUR up)
    groups: Optional[np.ndarray]    # uint32 per clause: the batch-wide index of its group's first clause (DISMAX up)
    ties: Optional[np.ndarray]      # float32 per clause: its group's tie, 0 outside a DisMax (DISMAX up)
    n_queries: int                  # the top-level queries: nodes 0 .. n_queries - 1


def _node_parts(q):
    """(clauses, float32 weights, occurs, mm) of one node as the device folds it: an Or's clauses all SHOULD, a Bool's
    as must, should, filter, must_not, a top-level DisMax as Bool(should=[it])."""
    if isinstance(q, DisMax):
        return [q], [np.float32(1.0)], [SA_OCCUR_SHOULD], 1
    if isinstance(q, Bool):
        cs, ws, os_ = q.occur_clauses()
        return cs, ws, os_, q.mm
    return q.clauses, q.weights, [SA_OCCUR_SHOULD] * len(q.clauses), q.mm


def _nodes(queries):
    """The nodes of a batch in flatten_bool's order: the queries, then each query's nested queries in pre-order
    (a sub-query object used twice is two nodes); and per node, the node indices of its nested clauses in order."""
    nodes, children = list(queries), [[] for _ in queries]

    def visit(n):
        for c in _node_parts(nodes[n])[0]:
            if isinstance(c, (Or, Bool)):
                nodes.append(c)
                children.append([])
                children[n].append(len(nodes) - 1)
                visit(len(nodes) - 1)
    for q in range(len(queries)):
        visit(q)
    return nodes, children


def flatten_bool(queries, form):
    """Boolean queries as sa_score_batch_topk_bool takes them, for a form at least that of every query (bool_form):
    a BoolBatch with only the arrays `form` reads, so a lighter form neither builds nor passes the others.

    OR_AND: Or / And queries, and plain ones (search_topk's terms and phrases) as one-clause nodes with mm 1; clauses,
    node_starts (one node per query) and mm.  OCCUR adds per clause float32 weights
    and uint8 SA_OCCUR_* roles: an Or's clauses all SHOULD, a Bool's as must, should, filter, must_not.  DISMAX expands
    each DisMax into its members (their own weights, the DisMax's role) and adds per clause groups and ties; a top-level
    DisMax is Bool(should=[it]).  NESTED adds the nested queries as nodes after the queries, each query's in pre-order
    (every child after its parent), and clause_node: a nested clause is None in `clauses`, with its node, its Boost's
    weight, its role and a group of its own.  A batch flattened for a heavier form than its own carries the lighter
    form's arrays unchanged, plus self-groups, zero ties and SA_NO_NODE."""
    queries = list(queries)
    clauses, starts, mm = [], [0], []
    if form == OR_AND:
        for q in queries:
            if isinstance(q, Or):
                clauses.extend(q.clauses)
                mm.append(q.mm)
            else:
                clauses.append(q)
                mm.append(1)
            starts.append(len(clauses))
        return BoolBatch(clauses, _u32(starts), None, _u32(mm), None, None, None, None, len(queries))
    nodes, children = _nodes(queries) if form == NESTED else (queries, None)
    weights, occurs, cnode, groups, ties = [], [], [], [], []
    zero = np.float32(0.0)
    for n, node in enumerate(nodes):
        cs, ws, os_, qmm = _node_parts(node)
        if form == OCCUR:
            clauses.extend(cs)
            weights.extend(ws)
            occurs.extend(os_)
        else:
            kids = iter(children[n]) if children else None
            for c, w, o in zip(cs, ws, os_):
                first = len(clauses)
                if isinstance(c, (Or, Bool)):
                    members, tie, child = [(None, w)], zero, next(kids)
                elif isinstance(c, DisMax):
                    members, tie, child = list(zip(c.clauses, c.weights)), c.tie, SA_NO_NODE
                else:
                    members, tie, child = [(c, w)], zero, SA_NO_NODE
                for m, mw in members:
                    clauses.append(m)
                    cnode.append(child)
                    weights.append(mw)
                    occurs.append(o)
                    groups.append(first)
                    ties.append(tie)
        starts.append(len(clauses))
        mm.append(qmm)
    dismax = form >= DISMAX
    return BoolBatch(clauses, _u32(starts), _u32(cnode) if form == NESTED else None, _u32(mm),
                     np.asarray(weights, dtype=np.float32), np.asarray(occurs, dtype=np.uint8),
                     _u32(groups) if dismax else None, np.asarray(ties, dtype=np.float32) if dismax else None,
                     len(queries))


def _u32(x):
    return np.asarray(x, dtype=np.uint32)


def dismax_members(queries):
    """Indices of the clauses that are DisMax members, into the clause list of flatten_bool for DISMAX or NESTED."""
    out, n = [], 0
    for q in _nodes(queries)[0]:
        for c in _top_clauses(q):
            k = len(c.clauses) if isinstance(c, DisMax) else 1
            if isinstance(c, DisMax):
                out.extend(range(n, n + k))
            n += k
    return out


def check_dismax_members(members, params):
    """ValueError unless every DisMax member can be ranked by its max: params(i) -> (k1, b, avgdl, idf) of member i
    must be sparse-safe (k1 > 0, 0 <= b < 1, finite idf >= 0), so that every weighted score is >= +0.  A member on a
    column whose avgdl is 0 scores 0 everywhere and is accepted.  members: (index, clause) pairs."""
    for i, c in members:
        k1, b, avgdl, idf = (np.float32(x) for x in params(i))
        if avgdl == 0:
            continue
        if not (np.isfinite(k1) and k1 > 0 and 0 <= b < 1 and np.isfinite(avgdl) and avgdl > 0 and np.isfinite(idf)
                and idf >= 0 and not np.signbit(idf)):
            raise ValueError(f"DisMax members need ordinary BM25 parameters (k1 > 0, 0 <= b < 1, finite idf >= 0): "
                             f"{c!r} has k1={float(k1)}, b={float(b)}, idf={float(idf)}")


def column_terms(clauses, feature_slot, facet_slot):
    """The Feature, Range and In leaves of a flattened clause list (BoolBatch.clauses) as the C entry points take
    them: {index: (clause entries, float32 parameter)} -- a Feature's reserved term id with its parameter, a Range's
    SA_RANGE_TERM and bound bits, an In's SA_IN_TERM and codes, the last two with parameter 0.  feature_slot(i, c) ->
    the slot of c's feature column on clause i's index; facet_slot(i, c) -> (slot, n_buckets) of c's facet column
    there; each raises ValueError for a name that is not set.  An In code >= n_buckets is a ValueError."""
    out = {}
    for i, c in enumerate(clauses):
        f = c.clause if isinstance(c, Field) else c
        if isinstance(f, Feature):
            out[i] = ([f.term_id(feature_slot(i, f))], f.param)
        elif isinstance(f, Range):
            out[i] = (f.entries(feature_slot(i, f)), np.float32(0))
        elif isinstance(f, In):
            slot, n_buckets = facet_slot(i, f)
            if max(f.codes) >= n_buckets:
                raise ValueError(f"{f!r}: codes are below facet {f.name!r}'s {n_buckets} buckets")
            out[i] = (f.entries(slot), np.float32(0))
    return out


def feature_terms(clauses, slot):
    """The feature leaves of a flattened clause list (BoolBatch.clauses) as the C entry points take them:
    {index: (reserved term id, float32 parameter)}.  slot(i, feature) -> the feature's slot on clause i's index (it
    raises ValueError for a name that is not set there).  column_terms restricted to Feature clauses."""
    only = [c if isinstance(c.clause if isinstance(c, Field) else c, Feature) else None for c in clauses]
    return {i: (e[0], p) for i, (e, p) in column_terms(only, slot, None).items()}


class Rescore:
    """Window rescoring, as Elasticsearch's `rescore` and Solr's `rq={!rerank}`: the `rescore=` argument of
    SearchArray.search_topk and solr.fields_topk.  Per query q, the call without `rescore` at k=window ranks the
    window (pass 1, with its `where=` and `facets=`; hits are pass 1's); s2 is queries[q] scored at the window's docs
    (SearchArray.score_docs / solr.fields_score_docs, with this slop); each doc's combined score is
    c = float32(query_weight * s1) + float32(rescore_weight * s2), each product rounded to float32, then the sum; and
    the result is the top k of the window by (c desc, id asc), with c as its scores and empty slots NO_DOC / 0.

    queries: one query per query of the call, of any form score_docs takes (Field clauses under fields_topk).  window:
    an int in [k, 1,024] (checked at the call).  Weights are rounded to float32 once and must be finite, with
    query_weight > 0 and rescore_weight >= 0, so that every c of a ranked doc is > 0 (ValueError otherwise)."""

    def __init__(self, queries, window=100, query_weight=1.0, rescore_weight=1.0, slop=0):
        self.queries = list(queries)
        if isinstance(window, bool) or not isinstance(window, (int, np.integer)):
            raise ValueError(f"a rescore window is an int in [k, {TOPK_MAX}], not {window!r}")
        self.window = int(window)
        for name, w in (("query_weight", query_weight), ("rescore_weight", rescore_weight)):
            if isinstance(w, bool) or not isinstance(w, (int, float, np.integer, np.floating)):
                raise ValueError(f"{name} is a finite number, not {w!r}")
            with np.errstate(over="ignore"):
                w32 = np.float32(w)
            if not (math.isfinite(float(w)) and np.isfinite(w32)):
                raise ValueError(f"{name} is finite (in float32), not {w!r}")
        self.query_weight, self.rescore_weight = np.float32(query_weight), np.float32(rescore_weight)
        if not self.query_weight > 0:
            raise ValueError(f"query_weight must be > 0, not {query_weight!r}")
        if not self.rescore_weight >= 0:
            raise ValueError(f"rescore_weight must be >= 0, not {rescore_weight!r}")
        self.slop = slop

    def check(self, n_queries, k):
        """ValueError unless there is one rescore query per query and k <= window <= TOPK_MAX."""
        if len(self.queries) != n_queries:
            raise ValueError(f"Rescore has {len(self.queries)} queries for a call of {n_queries}: one per query")
        if not k <= self.window <= TOPK_MAX:
            raise ValueError(f"a rescore window is in [k, {TOPK_MAX}] = [{k}, {TOPK_MAX}], not {self.window}")

    def __repr__(self):
        return (f"Rescore({self.queries!r}, window={self.window}, query_weight={float(self.query_weight)!r}, "
                f"rescore_weight={float(self.rescore_weight)!r}, slop={self.slop!r})")


def rescore_window(docs, s1, s2, query_weight, rescore_weight, k):
    """Rescore's combine and order on the host: per row, c = float32(query_weight * s1) + float32(rescore_weight * s2)
    over the window's docs (uint32 [Q, W], NO_DOC in empty slots, whose c is 0), and the first k by (c desc, id asc)
    from one argsort of the keys (c_bits << 32) | ~doc.  Returns (docs uint32 [Q, k], c float32 [Q, k])."""
    from ._lib import NO_DOC
    docs = np.asarray(docs, dtype=np.uint32)
    empty = docs == NO_DOC
    c = np.float32(query_weight) * np.asarray(s1, dtype=np.float32) + np.float32(rescore_weight) * np.asarray(
        s2, dtype=np.float32)
    c = np.where(empty, np.float32(0), c).astype(np.float32)
    # c >= +0 for every doc (s1 > 0, weights and s2 >= 0), so its bits order as it does; an empty slot's key is 0
    keys = (c.view(np.uint32).astype(np.uint64) << np.uint64(32)) | (~docs).astype(np.uint64)
    order = np.argsort(~keys, axis=1, kind="stable")[:, :k]
    return np.take_along_axis(docs, order, axis=1), np.take_along_axis(c, order, axis=1)


# The largest k of the batched top-k (search_topk, fields_topk, edismax_topk): SA_TOPK_DEEP_MAX of
# include/searcharray_b200.h.  Above 32 every tile keeps its exact top k (the deep collectors).
TOPK_MAX = 1024


def check_k(k, limit=TOPK_MAX):
    """k as an int, or ValueError unless 1 <= k <= limit: refused before any device work."""
    if isinstance(k, bool) or not isinstance(k, (int, np.integer)) or not 1 <= k <= limit:
        raise ValueError(f"k must be in [1, {limit}], not {k!r}")
    return int(k)
