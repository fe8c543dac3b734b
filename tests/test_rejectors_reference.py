"""Every correspondence rejector against a plain reference of its own list (CPU part).

The rules, from PCL's registration/src/correspondence_rejection_*.cpp, in numpy:

* DISTANCE: keep d < float(p) * float(p), the product and the comparison in float, strict; input order kept.
* MEDIAN: the median is element c // 2 of the ascending distances, as a double (-0.0 reported as +0.0); keep
  double(d) <= median * factor; input order kept.
* ONE_TO_ONE: drop index_match < 0; for each match keep the smallest (distance, input position); output in index_match
  order.
* TRIMMED: keep = max(floor(float(clamp01(p)) * float(n)) in float, uint32(min)), clamp01 as setOverlapRatio does
  (NaN gives 0); when keep < n the first keep entries of the stable sort by distance, otherwise the input unchanged.
* SURFACE_NORMAL: tests/test_consumers_reference.py (float dot product, kept when its double is > p).
* The chain inside the ICP loop: every stage sees the survivors of the one before in source-position order (so ties
  break by position even after a one-to-one), and the list the loop keeps is in that order.

Distances are any non-NaN float: -0.0 compares equal to +0.0, negatives come before zero, +inf after FLT_MAX.

The lists: the 1-NN correspondence lists of every scene of tests/test_search_reference.py (ungated, two gates, a
permuted index subset, reciprocal), and synthetic lists at the sizes around 0, a block and a radix tile, with
distances that tie, zeros of both signs, negatives, denormals, FLT_MAX and +inf, and matches that all hit one target,
are -1, or reach 2^31 - 1.  The oracle's stand-alone rejectors, its chains and its ICP loop are checked against the
reference here; the device in tests/test_gpu_rejectors_reference.py.  The teeth tests show that each rule the
reference fixes changes rows on these lists when it is replaced by its likeliest wrong twin."""
import os
import sys
from collections import Counter

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_search_reference as R  # noqa: E402
from test_consumers_reference import surface_normal_ref  # noqa: E402
from test_normals_reference import knn_sets  # noqa: E402

CORR_DTYPE = R.CORR_DTYPE
DISTANCE, MEDIAN, ONE_TO_ONE, TRIMMED, SURFACE_NORMAL = 0, 1, 2, 3, 4
FLT_MAX = float(np.finfo(np.float32).max)
MEDIAN_FACTORS = (0.0, 0.5, 1.0, 1.5, 3.0)
# (p, n) where floor(float(p) * float(n)) in float and floor(double(float(p)) * n) in double differ
FLOAT_KEEP_CASES = ((0.7, 10), (0.9, 1000), (0.9, 10))
SIZES = (0, 1, 2, 3, 4, 10, 255, 256, 257, 1000, 4095, 4096, 4097)
CHAIN4 = [(MEDIAN, 3.0, 0), (ONE_TO_ONE, 0.0, 0), (TRIMMED, 0.9, 100), (DISTANCE, 0.2, 0)]


# ---------------------------------------------------------------------------------------------------------------------
# the reference: each rule returns the rows of its input that survive, in output order
# ---------------------------------------------------------------------------------------------------------------------
def distance_limit(p):
    with np.errstate(over="ignore", invalid="ignore"):
        return np.float32(np.float32(p) * np.float32(p))


def sel_distance(d, p):
    return np.nonzero(d < distance_limit(p))[0]


def median_of(d):
    if d.size == 0:
        return 0.0
    return float(np.sort(d.astype(np.float64))[d.size // 2]) + 0.0


def sel_median(d, factor):
    med = median_of(d)
    with np.errstate(invalid="ignore"):
        return np.nonzero(d.astype(np.float64) <= med * float(factor))[0], med


def sel_one_to_one(m, d):
    pos = np.nonzero(m >= 0)[0]
    order = np.lexsort((pos, d[pos].astype(np.float64), m[pos]))
    s = pos[order]
    head = np.r_[True, m[s][1:] != m[s][:-1]] if s.size else np.zeros(0, bool)
    return s[head]


def overlap_clamp(p):
    r = np.float32(p)
    r = r if r > 0 else np.float32(0)          # std::max(0.0f, r): NaN gives 0
    return r if r < 1 else np.float32(1)       # std::min(1.0f, r)


def trimmed_keep(p, n, min_correspondences):
    k = int(np.floor(np.float32(overlap_clamp(p) * np.float32(n))))
    return max(k, int(min_correspondences) & 0xFFFFFFFF)


def sel_trimmed(d, p, min_correspondences):
    keep = trimmed_keep(p, d.size, min_correspondences)
    if keep >= d.size:
        return np.arange(d.size)
    return np.argsort(d.astype(np.float64), kind="stable")[:keep]


def reject_ref(c, kind, p=0.0, min_correspondences=0):
    """One stand-alone rejector: (remaining, median)."""
    d, m = c["distance"], c["index_match"]
    if kind == DISTANCE:
        return c[sel_distance(d, p)], 0.0
    if kind == MEDIAN:
        s, med = sel_median(d, p)
        return c[s], med
    if kind == ONE_TO_ONE:
        return c[sel_one_to_one(m, d)], 0.0
    assert kind == TRIMMED
    return c[sel_trimmed(d, p, min_correspondences)], 0.0


def chain_ref(c, chain, normals=None, tie_by_input_order=False):
    """The ICP loop's chain on a list in position order; normals = (source, target) for SURFACE_NORMAL.
    tie_by_input_order: the literal chain instead (each stage takes the previous one's output order), for the teeth."""
    for kind, p, mn in chain:
        if kind == SURFACE_NORMAL:
            c = surface_normal_ref(c, normals[0], normals[1], p)
            continue
        d, m = c["distance"], c["index_match"]
        s = (sel_distance(d, p) if kind == DISTANCE else sel_median(d, p)[0] if kind == MEDIAN else
             sel_one_to_one(m, d) if kind == ONE_TO_ONE else sel_trimmed(d, p, mn))
        c = c[s if tie_by_input_order else np.sort(s)]
    return c


# ---------------------------------------------------------------------------------------------------------------------
# the lists
# ---------------------------------------------------------------------------------------------------------------------
def corr(q, m, d):
    out = np.empty(len(d), CORR_DTYPE)
    out["index_query"], out["index_match"], out["distance"] = q, m, np.asarray(d, np.float32)
    return out


def synthetic_lists():
    """name -> list: every size of SIZES with several distance and match patterns."""
    rng = np.random.default_rng(61)
    special = np.array([0.0, -0.0, -1e-3, 2e-3, -2e-3, 1e-40, -1e-40, FLT_MAX, np.inf, 5e-4, 1e-45, 3e-3], np.float32)
    squares = (np.float32([0.1, 0.2, 0.3, 0.05]) * np.float32([0.1, 0.2, 0.3, 0.05])).astype(np.float32)
    out = {}
    for n in SIZES:
        q = np.arange(n, dtype=np.int32)
        m_rand = rng.integers(0, max(n // 3, 1), n).astype(np.int32)
        m_neg = np.where(np.arange(n) % 7 == 3, -1, m_rand).astype(np.int32)
        m_big = (2 ** 31 - 1 - rng.integers(0, max(n // 2, 1), n)).astype(np.int32)
        out[f"n={n} all equal, one target"] = corr(q, np.zeros(n, np.int32), np.full(n, 0.0025, np.float32))
        for levels in (2, 3, 6):
            d = (rng.integers(0, levels, n) + 1).astype(np.float32) * np.float32(1e-3)
            out[f"n={n} {levels} levels"] = corr(q, m_neg if levels == 3 else m_rand, d)
        out[f"n={n} zeros of both signs"] = corr(q, m_rand, np.where(rng.random(n) < 0.5, -0.0, 0.0).astype(np.float32))
        out[f"n={n} special values"] = corr(q, m_neg, special[rng.integers(0, special.size, n)])
        out[f"n={n} squares, large ids"] = corr(q, m_big, squares[rng.integers(0, squares.size, n)])
        out[f"n={n} random"] = corr(q, m_rand, (rng.random(n, dtype=np.float32) ** 2).astype(np.float32))
    return out


SYNTH = synthetic_lists()


def scene_lists(name):
    """The 1-NN lists of one scene's queries (R.make_queries), through R.corr_ref: ungated, two gates, a permuted index
    subset and reciprocal."""
    pts, spacing = R.SCENES[name]()
    cloud = R.xyz1(pts)
    q, _ = R.make_queries(name, pts, spacing, n_jitter=6_000, n_boundary=2_000, n_beyond=200)
    q = R.xyz1(q)
    nn, nd = knn_sets(cloud, q, 1, return_d2=True)
    nn, nd = nn[:, 0], nd[:, 0]
    ind = np.random.default_rng(5).permutation(q.shape[0])[: q.shape[0] // 3].astype(np.int32)
    return {
        f"{name} ungated": R.corr_ref(nn, nd),
        f"{name} gate 3 spacings": R.corr_ref(nn, nd, 3 * spacing),
        f"{name} gate 0.3 spacings": R.corr_ref(nn, nd, 0.3 * spacing),
        f"{name} permuted subset": R.corr_ref(nn, nd, spacing, indices=ind),
        f"{name} reciprocal": R.corr_ref(nn, nd, 3 * spacing, back=R.reciprocal_back(q, cloud)),
    }


def params_for(c):
    """(kind, p, min) of every stand-alone check of list c."""
    n = c.size
    d = np.sort(c["distance"].astype(np.float64))
    out = [(ONE_TO_ONE, 0.0, 0)]
    fin = d[np.isfinite(d) & (d > 0)]
    limits = [0.0, 1.0, 0.05, 0.1, 0.3, FLT_MAX]
    if fin.size:
        limits += [float(np.sqrt(fin[fin.size // 2])), float(np.sqrt(fin[-1]))]
    out += [(DISTANCE, p, 0) for p in limits]
    out += [(MEDIAN, f, 0) for f in MEDIAN_FACTORS]
    out += [(TRIMMED, 0.0, k) for k in {0, 1, max(n - 1, 0), n, n + 1}]
    out += [(TRIMMED, p, 0) for p in (0.5, 0.7, 0.9, 1.0, -0.5, 1.5, float("nan"))]
    out += [(TRIMMED, 0.5, -1), (TRIMMED, 0.5, 3_000_000_000), (TRIMMED, 0.3, 2)]
    return out


# ---------------------------------------------------------------------------------------------------------------------
# the oracle against the reference
# ---------------------------------------------------------------------------------------------------------------------
def _same(got, want):
    return got.size == want.size and got.tobytes() == want.tobytes()


KIND_NAMES = ("distance", "median", "one-to-one", "trimmed")


def check_standalone(reject, lists):
    """reject(c, kind, p, min) -> (remaining, median) against the reference on every list and parameter; fails with
    every (list, rejector) that differs."""
    checked, bad, by_rule, by_list = 0, [], Counter(), Counter()
    for name, c in lists.items():
        for kind, p, mn in params_for(c):
            got, gmed = reject(c, kind, p, mn)
            want, wmed = reject_ref(c, kind, p, mn)
            rule = f"{KIND_NAMES[kind]} p={p:.6g} min={mn}"
            if not _same(got, want):
                bad.append(f"{name}: {rule}: {got.size} kept, the reference keeps {want.size}")
            elif kind == MEDIAN and np.float64(gmed).tobytes() != np.float64(wmed).tobytes():
                bad.append(f"{name}: {rule}: median {gmed!r}, the reference's {wmed!r}")
            else:
                rule = None
            if rule:
                by_rule[rule if kind in (TRIMMED, MEDIAN) else KIND_NAMES[kind]] += 1
                by_list[name.split(" ", 1)[-1]] += 1
            checked += 1
    assert not bad, (f"{len(bad)} of {checked} differ\nby rejector: {dict(by_rule)}\nby list: {dict(by_list)}\n"
                     + "\n".join(bad[:20]))
    return checked


CHAINS = {
    "one-to-one, trimmed": [(ONE_TO_ONE, 0.0, 0), (TRIMMED, 0.6, 0)],
    "trimmed, one-to-one": [(TRIMMED, 0.6, 0), (ONE_TO_ONE, 0.0, 0)],
    "chain of four": CHAIN4,
    "median, one-to-one, trimmed to c - 1": [(MEDIAN, 1.5, 0), (ONE_TO_ONE, 0.0, 0), (TRIMMED, 0.999, 0)],
}


def test_oracle_standalone_synthetic(orc):
    """Every synthetic list, every parameter: the oracle's records, their order and its median."""
    n = check_standalone(lambda c, k, p, m: orc.reject(c, k, p=p, min_correspondences=m), SYNTH)
    assert n > 1000


@pytest.mark.parametrize("name", list(R.SCENES))
def test_oracle_standalone_scene_lists(orc, name):
    lists = scene_lists(name)
    assert all(c.size > 0 for c in lists.values()), {k: c.size for k, c in lists.items()}
    check_standalone(lambda c, k, p, m: orc.reject(c, k, p=p, min_correspondences=m), lists)
    for cname, chain in CHAINS.items():
        for lname, c in lists.items():
            assert _same(orc.reject_chain(c, chain)[0], chain_ref(c, chain)), (lname, cname)


def test_oracle_chains_synthetic(orc):
    """Chains of stand-alone calls (each stage takes the previous one's output as it comes) and the loop's chain
    (each stage sees position order)."""
    for name, c in SYNTH.items():
        for cname, chain in CHAINS.items():
            lit = c
            for kind, p, mn in chain:
                lit = orc.reject(lit, kind, p=p, min_correspondences=mn)[0]
            assert _same(lit, chain_ref(c, chain, tie_by_input_order=True)), (name, cname)
            assert _same(orc.reject_chain(c, chain)[0], chain_ref(c, chain)), (name, cname)


def test_trimmed_count_past_float_precision():
    """n = 2^24 + 5: float(n) rounds to 2^24 + 4, so overlap 1.0 still trims one entry, as PCL's float count does."""
    n = 2 ** 24 + 5
    assert trimmed_keep(1.0, n, 0) == n - 1
    assert trimmed_keep(1.5, n, 0) == n - 1 and trimmed_keep(-0.5, n, 7) == 7 and trimmed_keep(float("nan"), n, 0) == 0
    assert trimmed_keep(0.5, 10, -1) == 2 ** 32 - 1 and trimmed_keep(0.5, 10, 3_000_000_000) == 3_000_000_000


# ---------------------------------------------------------------------------------------------------------------------
# the oracle's ICP loop against the reference chain
# ---------------------------------------------------------------------------------------------------------------------
def lattice_pair():
    """Target: the 40 x 40 x 6 lattice of spacing 1/32; source: the lattice of spacing 1/64 inside it, shifted by one
    fine step along x.  Every 1-NN distance is one of a few exact values and most targets are the nearest point of
    several sources at the same distance, so the first iteration is full of exact ties.  The source comes in a seeded
    random order, so position order and target order differ."""
    h = 1.0 / 32
    g = np.stack(np.meshgrid(np.arange(40), np.arange(40), np.arange(6), indexing="ij"), -1).reshape(-1, 3)
    tgt = (g * h).astype(np.float32)
    fg = np.stack(np.meshgrid(np.arange(4, 74), np.arange(4, 74), np.arange(2, 9), indexing="ij"), -1).reshape(-1, 3)
    src = (fg * (h / 2) + [h / 2, 0, 0]).astype(np.float32)
    return tgt, src[np.random.default_rng(29).permutation(src.shape[0])]


LOOP_CHAINS = {
    "one-to-one, trimmed": [(ONE_TO_ONE, 0.0, 0), (TRIMMED, 0.6, 0)],
    "trimmed, one-to-one": [(TRIMMED, 0.6, 0), (ONE_TO_ONE, 0.0, 0)],
    "chain of four": CHAIN4,
    "median": [(MEDIAN, 1.0, 0)],
}


@pytest.mark.parametrize("chain", list(LOOP_CHAINS))
def test_oracle_loop_list_on_the_lattice(orc, chain):
    """The oracle's list after the chain in its first ICP iteration equals the reference chain on the reference 1-NN
    list of the lattice pair: the same pairs, in source-position order."""
    tgt, src = lattice_pair()
    T, S = R.xyz1(tgt), R.xyz1(src)
    nn, nd = knn_sets(T, S, 1, return_d2=True)
    want = chain_ref(R.corr_ref(nn[:, 0], nd[:, 0]), LOOP_CHAINS[chain])
    o = orc.icp_align_rejectors(S, T, LOOP_CHAINS[chain], max_iterations=1, nthreads=4)
    got = o["correspondences"]
    assert o["n_correspondences"] == want.size
    assert np.array_equal(np.sort(got["index_query"]), want["index_query"]), (chain, got.size, want.size)
    assert _same(got, want), chain


# ---------------------------------------------------------------------------------------------------------------------
# teeth: each rule, replaced by its likeliest wrong twin, changes rows on the lists above
# ---------------------------------------------------------------------------------------------------------------------
def _changes(rule, twin, lists):
    return [name for name, c in lists.items() if not _same(rule(c), twin(c))]


def test_teeth_tie_rule_after_one_to_one():
    """[ONE_TO_ONE, TRIMMED]: position order against the one-to-one's index_match order, on the lattice pair and on
    the synthetic lists."""
    chain = LOOP_CHAINS["one-to-one, trimmed"]
    tgt, src = lattice_pair()
    nn, nd = knn_sets(R.xyz1(tgt), R.xyz1(src), 1, return_d2=True)
    lat = {"lattice": R.corr_ref(nn[:, 0], nd[:, 0])}
    def kept(c, literal):  # the pairs kept, whatever their order
        return np.sort(chain_ref(c, chain, tie_by_input_order=literal)["index_query"])
    for lists in (lat, SYNTH):
        assert _changes(lambda c: kept(c, False), lambda c: kept(c, True), lists)


def test_teeth_median_index():
    twin = lambda c: c[np.nonzero(c["distance"].astype(np.float64) <= (float(np.sort(  # noqa: E731
        c["distance"].astype(np.float64))[(c.size - 1) // 2]) if c.size else 0.0))[0]]
    assert _changes(lambda c: reject_ref(c, MEDIAN, 1.0)[0], twin, SYNTH)


def test_teeth_float_keep_count():
    """floor(float(p) * float(n)) in float against the same product in double."""
    for p, n in FLOAT_KEEP_CASES:
        assert trimmed_keep(p, n, 0) != int(np.floor(np.float64(np.float32(p)) * n)), (p, n)
    lists = {f"n={n}": SYNTH["n=4097 random"][:n] for n in (10, 1000)}

    def twin(c, p):
        keep = int(np.floor(np.float64(np.float32(p)) * c.size))
        return c[np.argsort(c["distance"].astype(np.float64), kind="stable")[:keep]] if keep < c.size else c
    changed = [(name, p) for p in (0.7, 0.9) for name, c in lists.items()
               if not _same(reject_ref(c, TRIMMED, p)[0], twin(c, p))]
    assert changed


def test_teeth_distance_limit_precision_and_strictness():
    """DISTANCE: float(p)^2 in float against p^2 in double, and < against <=."""
    rng = np.random.default_rng(3)
    ps = rng.random(4000) * 0.3
    d = np.array([np.nextafter(distance_limit(p), np.float32(0)) for p in ps], np.float32)
    flips = np.nonzero((d < distance_limit(ps).astype(np.float32)) != (d.astype(np.float64) < ps * ps))[0]
    assert flips.size, "no p whose float square and double square straddle a float"
    c = corr(np.arange(flips.size), np.arange(flips.size), d[flips])
    lists = {"near the float square": c}
    for p in ps[flips][:5]:
        assert _changes(lambda x: reject_ref(x, DISTANCE, p)[0],
                        lambda x: x[np.nonzero(x["distance"].astype(np.float64) < p * p)[0]], lists), p
    eq = {k: v for k, v in SYNTH.items() if "squares" in k}
    assert _changes(lambda x: reject_ref(x, DISTANCE, 0.2)[0],
                    lambda x: x[np.nonzero(x["distance"] <= distance_limit(0.2))[0]], eq)


def test_teeth_signed_zero_and_negative_order():
    """The rules order -0.0 with +0.0 and negatives before zero; an order of the raw bit patterns (what an unsigned
    radix key of the bits gives) changes rows."""
    def bits_rank(c):
        return c["distance"].view(np.uint32).astype(np.int64)
    lists = {k: v for k, v in SYNTH.items() if "signs" in k or "special" in k}
    twin = lambda c: c[np.argsort(bits_rank(c), kind="stable")[:trimmed_keep(0.5, c.size, 0)]]  # noqa: E731
    assert _changes(lambda c: reject_ref(c, TRIMMED, 0.5)[0], twin, lists)
