"""The device ICP loop's decisions against the reference of tests/test_loop_reference.py, step by step and at the stop:
state, converged, iterations and final transformation bit for bit, the MSE against PCL's summation order, thresholds
set to recorded values, the less used criteria, the batch forms, and the previous MSE that a session carries from one
align to the next.  Needs an H100: run with -m gpu."""
import os
import sys
import time
from collections import defaultdict

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_loop_reference as L  # noqa: E402
import test_rejectors_reference as RR  # noqa: E402

pytestmark = pytest.mark.gpu

COUNT = defaultdict(int)
T0 = [0.0]
K = 10
SCENES = ("synthetic pair", "lattice", "map_1e5")
ESTIMATORS = {"svd": (0, 0), "svd correlation": (0, 1), "point-to-plane": (1, 0), "symmetric": (2, 0)}
# the lattice's k-NN normals are all one plane (singular normal equations); the map scene runs the SVD
RUNS = [(s, e) for s in SCENES for e in ESTIMATORS if s == "synthetic pair" or e.startswith("svd")]
OFF = dict(transformation_epsilon=-1.0, euclidean_fitness_epsilon=-L.DBL_MAX, mse_threshold_absolute=0.0)


@pytest.fixture(scope="module")
def gpu():
    import pcl_b200
    pcl_b200.lib()
    ctx = pcl_b200.Context(0)
    T0[0] = time.time()
    yield pcl_b200, ctx
    ctx.close()
    print("\n" + "\n".join(f"{k:56s} {v:8d}" for k, v in sorted(COUNT.items())))
    print(f"test_gpu_loop_reference.py: {time.time() - T0[0]:.1f} s")


_SCENES = {}


def scene(orc, name):
    if name not in _SCENES:
        if name == "map_1e5":
            from test_gpu_search_reference import _icp_pair
            tgt, src, gate = _icp_pair(name)
            _SCENES[name] = (L._recs(orc, src), L._recs(orc, tgt), gate)
        else:
            _SCENES[name] = L.oracle_scene(orc, name)
    return _SCENES[name]


class Run:
    """One device session on a scene: records (8 floats: xyz 1 | normal 0), its index, the estimator."""

    def __init__(self, P, ctx, orc, name, est, dbl):
        self.P, self.ctx = P, ctx
        self.src, self.tgt, self.gate = scene(orc, name)
        self.e, self.no_u = ESTIMATORS[est]
        self.dbl = dbl
        self.scalar = np.float64 if dbl else np.float32
        self.index = P.Index(ctx, np.ascontiguousarray(self.tgt[:, :4]))
        self.tn = np.ascontiguousarray(self.tgt[:, 4:8])

    def kw(self, **crit):
        d = dict(max_iterations=K, max_correspondence_distance=self.gate, estimator=self.e, svd_no_umeyama=self.no_u,
                 scalar_is_double=int(self.dbl), with_normals_transform=int(self.e != 0))
        d.update(crit)
        return d

    def session(self, **crit):
        s = self.P.Icp(self.ctx, **self.kw(**crit))
        s.set_target(self.index, normals=self.tn)
        return s

    def set_source(self, s, guess=None, src=None):
        src = self.src if src is None else src
        s.set_source(np.ascontiguousarray(src[:, :4]), normals=np.ascontiguousarray(src[:, 4:8]) if self.e else None,
                     guess=guess)

    def record(self, guess=None, src=None, steps=K, **crit):
        """criteria off: [(n_pairs, last, mse)] and the pair lists, one per iteration"""
        s = self.session(**{**OFF, **crit})
        self.set_source(s, guess, src)
        out, lists = [], []
        for _ in range(steps):
            st = s.iterate(1)
            lists.append(s.get_correspondences())
            if st["state"] == L.NO_CORRESPONDENCES:
                out.append((st["n_correspondences"], np.eye(4), 0.0))
                break
            out.append((st["n_correspondences"], st["last"], st["mse"]))
            if st["state"] != L.NOT_CONVERGED:
                break
        s.close()
        return out, lists


def _params(kw):
    return L.params(max_iterations=kw.get("max_iterations", K), failure_after_max_iter=kw.get("failure_after_max_iter", 0),
                    max_iterations_similar=kw.get("max_iterations_similar_transforms", 0),
                    rot_eps=kw.get("transformation_rotation_epsilon", 0.0), trans_eps=kw["transformation_epsilon"],
                    rel_mse=kw["euclidean_fitness_epsilon"], abs_mse=kw["mse_threshold_absolute"])


def _check_stop(st, want, what):
    w = want[-1]
    assert (st["iterations"], st["state"], st["converged"]) == (w[2], w[0], w[1]), (what, st["iterations"], st["state"], w[:4])
    assert L.same_bits(st["final"], w[5]), (what, st["final"], w[5])


def criteria_settings(steps, scalar):
    """each criterion at recorded values and their neighbouring doubles, the similar counts at quantiles of the recorded
    values, failure_after_max_iter and max_iterations 0 and 1"""
    out = L.threshold_settings(steps, scalar)
    v = L._values(steps, scalar)
    for ms in (1, 2, 3):
        for q in (0.3, 0.6):
            if v["abs"]:
                out.append({**OFF, "mse_threshold_absolute": float(np.quantile(v["abs"], q)),
                            "max_iterations_similar_transforms": ms})
            if v["rel"]:
                out.append({**OFF, "euclidean_fitness_epsilon": float(np.quantile(v["rel"], q)),
                            "max_iterations_similar_transforms": ms})
            out.append({**OFF, "transformation_epsilon": float(np.quantile(v["t2"], q)),
                        "transformation_rotation_epsilon": -1.0, "max_iterations_similar_transforms": ms})
    n = len(steps)
    for fail in (0, 1):
        # a TRANSFORM that fires exactly at max_iterations, and one that does not fire
        t2_last = v["t2"][n - 1]
        out.append({**OFF, "max_iterations": n, "failure_after_max_iter": fail, "transformation_epsilon": t2_last,
                    "transformation_rotation_epsilon": -1.0})
        out.append({**OFF, "max_iterations": n, "failure_after_max_iter": fail})
    for mi in (0, 1):
        out.append({**OFF, "max_iterations": mi})
        out.append({**OFF, "max_iterations": mi, "failure_after_max_iter": 1, "mse_threshold_absolute": 1.0})
    out.append(dict(transformation_epsilon=0.0, euclidean_fitness_epsilon=-L.DBL_MAX, mse_threshold_absolute=1e-12))
    return out


@pytest.mark.parametrize("dbl", [False, True], ids=["float", "double"])
@pytest.mark.parametrize("name,est", RUNS)
def test_loop_steps_and_stops(gpu, orc, name, est, dbl):
    """Record the criteria-off run; then, for every setting, step the loop with iterate(1) and check every iteration's
    state, converged, iterations and final bits against the reference fed the device's own T_k and MSE; iterate() in
    one call and icp_align reach the same stats.  The MSE against pcl_mse of the iteration's pair list."""
    P, ctx = gpu
    r = Run(P, ctx, orc, name, est, dbl)
    steps, lists = r.record()
    assert len(steps) == K and all(n >= 3 for n, _, _ in steps)
    _check_mse(steps, lists, name)
    settings = criteria_settings(steps, r.scalar)
    if not dbl:
        # float Scalar: some recorded step has float and double evaluations of cos or t^2 that differ, and a threshold
        # between them must give the float answer
        split = [(k, L.cos_t2(T, np.float32), L.cos_t2(T, np.float32, ("cos, t^2 in double",))) for k, (_, T, _) in
                 enumerate(steps)]
        split = [x for x in split if x[1] != x[2]]
        assert split, name
        k, (cf, tf), (cd, td) = split[0]
        if tf != td:
            settings.append({**OFF, "transformation_epsilon": min(tf, td), "transformation_rotation_epsilon": -1.0})
        if cf != cd:
            settings.append({**OFF, "transformation_epsilon": 1.0, "transformation_rotation_epsilon": max(cf, cd)})
        COUNT["float runs with a float / double split"] += 1
    stops = set()
    for i, kw in enumerate(settings):
        p = _params(kw)
        s = r.session(**kw)
        r.set_source(s)
        ref = L.Criteria()
        L.start_align(ref, p)
        final = np.eye(4)
        it = 0
        while True:
            st = s.iterate(1)
            n_pairs, T_k, mse = (st["n_correspondences"], st["last"], st["mse"])
            if n_pairs < 3:
                ref.state = L.NO_CORRESPONDENCES
                want = (L.NO_CORRESPONDENCES, False, it)
            else:
                assert L.same_bits(T_k, steps[it][1]) and L.same_bits(mse, steps[it][2]), (name, kw, it)
                final = L.compose(T_k, final, r.scalar)
                it += 1
                conv = L.criteria_step(ref, p, r.scalar, it, T_k, mse)
                want = (ref.state, conv, it)
            assert (st["state"], st["converged"], st["iterations"]) == want, (name, est, kw, it, st["state"], want)
            assert L.same_bits(st["final"], final), (name, kw, it)
            COUNT["loop steps compared"] += 1
            if ref.state != L.NOT_CONVERGED:
                break
            assert it < K + 1
        s.close()
        stops.add((st["iterations"], st["state"]))
        COUNT["loop stops compared"] += 1
        if i % 7 == 0:
            s2 = r.session(**kw)
            r.set_source(s2)
            one = s2.iterate()
            s2.close()
            al = P.icp_align(ctx, np.ascontiguousarray(r.src[:, :4]), r.index,
                             src_normals=np.ascontiguousarray(r.src[:, 4:8]) if r.e else None, tgt_normals=r.tn,
                             **r.kw(**kw))
            for x in (one, al):
                assert (x["state"], x["converged"], x["iterations"]) == (st["state"], st["converged"], st["iterations"])
                assert x["final"].tobytes() == st["final"].tobytes()
            COUNT["iterate() / icp_align stops compared"] += 2
    print(f"\n{name}, {est}, {'double' if dbl else 'float'}: {len(settings)} settings, stops {sorted(stops)}")
    assert len(stops) >= 4


def _check_mse(steps, lists, name):
    """The device's MSE against calculateMSE's sequential sum: bit for bit when every summation order is exact (all
    distances multiples of the smallest ulp among them, q, and the sum below 2^53 q); otherwise each of the two sums
    lies within (n - 1) 2^-53 sum of the exact one, so the two MSEs within twice that over n (and a rounding each)."""
    for (n, _, mse), c in zip(steps, lists):
        d = c["distance"].astype(np.float64)
        assert d.size == n
        want = L.pcl_mse(c["distance"])
        nz = d[d > 0]
        q = float(np.min(np.spacing(nz.astype(np.float32)).astype(np.float64))) if nz.size else 1.0
        exact = nz.size == 0 or (np.all(np.mod(d, q) == 0) and d.sum() < 2.0 ** 53 * q)
        if exact:
            assert mse == want, (name, mse, want)
            COUNT[f"MSE checks exact ({name})"] += 1
        else:
            assert abs(mse - want) <= 2 * (n - 1) * 2.0 ** -53 * d.sum() / n + 2 * np.spacing(want), (name, mse, want)
            COUNT[f"MSE checks within the round-off bound ({name})"] += 1


def test_mse_decisions_outside_the_band(gpu, orc):
    """PCL's MSE and the device's could only decide an MSE test differently when the threshold lies within the
    round-off band of the difference; count the recorded steps inside the band, and check no decision differs outside."""
    P, ctx = gpu
    inside = differ = 0
    for name in ("synthetic pair", "map_1e5"):
        r = Run(P, ctx, orc, name, "svd", False)
        steps, lists = r.record()
        pcl = [L.pcl_mse(c["distance"]) for c in lists]
        dev = [m for _, _, m in steps]
        sums = [float(np.sum(c["distance"].astype(np.float64))) for c in lists]
        for k in range(1, len(steps)):
            band = 2 * (lists[k].size + lists[k - 1].size) * 2.0 ** -53 * (sums[k] / lists[k].size + sums[k - 1] / lists[k - 1].size)
            for thr in L._nb(abs(dev[k] - dev[k - 1])) + [abs(dev[k] - dev[k - 1]) * f for f in (0.5, 2.0)]:
                a, b = abs(dev[k] - dev[k - 1]) < thr, abs(pcl[k] - pcl[k - 1]) < thr
                if abs(thr - abs(dev[k] - dev[k - 1])) <= band:
                    inside += 1
                else:
                    differ += a != b
    print(f"\nMSE decisions: {inside} threshold settings inside the round-off band, {differ} differing outside")
    COUNT["MSE decisions inside the round-off band"] += inside
    assert differ == 0


def test_no_correspondences(gpu, orc):
    """Fewer than 3 pairs at iteration 1 (the rejector chain that keeps 2): NO_CORRESPONDENCES, converged = false, no
    iteration counted and the final transformation untouched.  A later NO_CORRESPONDENCES is in the host-compiled
    sequences of tests/test_loop_reference.py."""
    P, ctx = gpu
    r = Run(P, ctx, orc, "synthetic pair", "svd", False)
    s = r.session(**OFF)
    s.set_rejectors([(RR.ONE_TO_ONE, 0.0, 0), (RR.TRIMMED, 0.0, 2)])
    r.set_source(s)
    st = s.iterate()
    assert (st["state"], st["converged"], st["iterations"]) == (L.NO_CORRESPONDENCES, False, 0)
    assert st["final"].tobytes() == np.eye(4).tobytes()
    s.close()
    COUNT["NO_CORRESPONDENCES stops compared"] += 1


def _motions(r, B):
    rng = np.random.default_rng(5)
    out = [np.eye(4)]
    for b in range(1, B):
        T = L._rot(rng.normal(size=3), 0.01 * b)
        T[:3, 3] = rng.normal(size=3) * 0.002 * b
        out.append(T)
    return out


@pytest.mark.parametrize("targets", ["one target", "per-problem targets"])
def test_batch_against_reference(gpu, orc, targets):
    """iterate_batch: every problem stops where the reference of its own records says (a new criteria state each),
    under criteria that make the problems stop at different iterations."""
    P, ctx = gpu
    r = Run(P, ctx, orc, "synthetic pair", "svd", False)
    B = 6
    guesses = _motions(r, B)
    recs = [r.record(guess=g)[0] for g in guesses]
    stops = set()
    for kw in ({**OFF, "mse_threshold_absolute": float(np.quantile(L._values(recs[2], np.float32)["abs"], 0.5))},
               {**OFF, "euclidean_fitness_epsilon": 1e-3},
               {**OFF, "transformation_epsilon": float(np.quantile(L._values(recs[3], np.float32)["t2"], 0.5)),
                "transformation_rotation_epsilon": -1.0}):
        s = r.session(**kw)
        if targets != "one target":
            s.set_target_batch([r.index] * B)
        src = np.concatenate([r.src[:, :4]] * B)
        s.set_source_batch(np.ascontiguousarray(src), np.arange(B + 1) * r.src.shape[0], guesses=np.stack(guesses))
        got = s.iterate_batch()
        s.close()
        for p in range(B):
            want = L.loop_reference(L.Criteria(), _params(kw), np.float32, recs[p], final0=guesses[p])
            _check_stop(got[p], want, (targets, kw, p))
            stops.add((str(kw), got[p]["iterations"]))
            COUNT["batch problem stops compared"] += 1
    assert any(len({it for k2, it in stops if k2 == k}) >= 2 for k, _ in stops), stops


def test_prev_mse_carried_across_aligns(gpu, orc):
    """A session aligned again after set_source (the same source from guess = final, and another source) stops where
    the reference with the criteria state carried over says; the carried previous MSE decides the stop (the reference
    that resets it predicts another).  pclb200_icp_align and set_source_batch start from a new criteria state."""
    P, ctx = gpu
    for est in ("svd", "point-to-plane"):
        for dbl in (False, True):
            r = Run(P, ctx, orc, "synthetic pair", est, dbl)
            kw = {**OFF, "mse_threshold_absolute": 1.0}   # every MSE lies in [0, gate^2]
            p = _params(kw)
            s = r.session(**kw)
            r.set_source(s)
            first = s.iterate()
            rec1, _ = r.record()
            ref = L.Criteria()
            want1 = L.loop_reference(ref, p, r.scalar, rec1)
            _check_stop(first, want1, "first align")
            other = r.src.copy()
            other[:, :3] += np.float32([0.003, -0.002, 0.001])
            for label, src, guess in (("same source, guess = final", None, first["final"]), ("another source", other, None)):
                carried = L.Criteria()
                carried.prev_mse = ref.prev_mse
                r.set_source(s, guess=guess, src=src)
                got = s.iterate()
                rec, _ = r.record(guess=guess, src=src)
                want = L.loop_reference(carried, p, r.scalar, rec, final0=guess)
                _check_stop(got, want, (est, dbl, label))
                fresh = L.loop_reference(L.Criteria(), p, r.scalar, rec, final0=guess)
                assert L.stop_of(fresh)[:2] != L.stop_of(want)[:2], (label, L.stop_of(fresh)[:2])
                ref = carried
                COUNT["across-align stops compared"] += 1
            # the one-call align and a batch after these aligns start fresh
            al = P.icp_align(ctx, np.ascontiguousarray(r.src[:, :4]), r.index,
                             src_normals=np.ascontiguousarray(r.src[:, 4:8]) if r.e else None, tgt_normals=r.tn,
                             guess=first["final"], **r.kw(**kw))
            rec, _ = r.record(guess=first["final"])
            _check_stop(al, L.loop_reference(L.Criteria(), p, r.scalar, rec, final0=first["final"]), "icp_align")
            if r.e == 0:
                s.set_source_batch(np.ascontiguousarray(r.src[:, :4]), [0, r.src.shape[0]],
                                   guesses=first["final"][None])
                b = s.iterate_batch()[0]
                _check_stop(b, L.loop_reference(L.Criteria(), p, r.scalar, rec, final0=first["final"]), "batch")
                assert b["iterations"] == 2
            s.close()
