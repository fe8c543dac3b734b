"""The ICP loop's decisions against a plain reference of PCL's source (CPU part).

What decides when the loop stops and what the caller gets back, restated in numpy line by line:

* ``criteria_step``: DefaultConvergenceCriteria::hasConverged (impl/default_convergence_criteria.hpp:49-140).  The reset
  at the top; ``iterations >= max_iterations`` (FAILURE_AFTER_MAX_ITERATIONS carries on to the other tests); the cosine
  ``0.5 * double(((T00 + T11) + T22) - 1)`` and ``t^2 = ((t0 t0 + t1 t1) + t2 t2)`` evaluated in Scalar, then widened;
  ``>=`` on the rotation test, ``<=`` on the translation test, strict ``<`` on both MSE tests; one similar-count
  increment per iteration, a reset when nothing was similar; the previous MSE written only when no criterion fired.
  The rotation threshold is set only by an epsilon > 0 (icp.hpp:160-161); otherwise the object keeps the one it had.
* ``loop_reference``: the do-while of icp.hpp:164-241 around it.  Fewer than 3 pairs stop with NO_CORRESPONDENCES and
  converged = false, before any composition or count; otherwise ``final = T_k * final`` in Scalar, coefficient by
  coefficient in Eigen's order ``((a0 b0 + a1 b1) + a2 b2) + a3 b3``, then ``++iterations``, then the criteria.
* The criteria object outlives one align (icp.h:155): a second align starts from the previous MSE the first one left.
* ``pcl_mse``: calculateMSE (default_convergence_criteria.h:262-269), a sequential fp64 sum in list order over n.

Checked here: the device's criteria and composition compiled for the host (tests/host/loop_host_test.cpp) on seeded and
hand-made sequences, bit for bit; the oracle's loop on recorded ICP runs with thresholds set to recorded values and
their neighbouring doubles; and that each likely slip of the rules changes at least one predicted stop.  The device
loop itself: tests/test_gpu_loop_reference.py."""
import math
import os
import shutil
import struct
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

DBL_MAX = float(np.finfo(np.float64).max)
NOT_CONVERGED, ITERATIONS, TRANSFORM, ABS_MSE, REL_MSE, NO_CORRESPONDENCES, FAILURE_AFTER_MAX_ITERATIONS = range(7)
# the likely slips of the rules; each must change a predicted stop somewhere (test_teeth)
SLIPS = ("abs <=", "rel <=", "translation <", "cos, t^2 in double", "similar count not reset",
         "prev_mse on the converging iteration", "prev_mse reset per align", "final * T_k", "composition in double")


class Criteria:
    """The members of DefaultConvergenceCriteria that outlive one align (default_convergence_criteria.h:263-321)."""

    def __init__(self):
        self.state = NOT_CONVERGED
        self.similar = 0
        self.prev_mse = DBL_MAX
        self.rotation_threshold = 0.99999


def params(max_iterations=10, failure_after_max_iter=False, max_iterations_similar=0, rot_eps=0.0, trans_eps=0.0,
           rel_mse=-DBL_MAX, abs_mse=1e-12):
    return dict(max_iterations=max_iterations, failure_after_max_iter=bool(failure_after_max_iter),
                max_iterations_similar=max_iterations_similar, rot_eps=float(rot_eps), trans_eps=float(trans_eps),
                rel_mse=float(rel_mse), abs_mse=float(abs_mse))


def cos_t2(T, scalar, slip=()):
    """(cos_angle, translation_sqr) as hasConverged evaluates them: in Scalar, then widened."""
    S = np.float64 if (scalar == np.float64 or "cos, t^2 in double" in slip) else np.float32
    t = np.asarray(T, dtype=np.float64).reshape(4, 4).astype(S)
    cos = 0.5 * float(((t[0, 0] + t[1, 1]) + t[2, 2]) - S(1))
    t2 = float((t[0, 3] * t[0, 3] + t[1, 3] * t[1, 3]) + t[2, 3] * t[2, 3])
    return cos, t2


def criteria_step(state, p, scalar, iterations, T_k, mse, slip=()):
    """DefaultConvergenceCriteria::hasConverged; returns converged and updates state."""
    if state.state != NOT_CONVERGED:
        state.similar = 0
        state.state = NOT_CONVERGED
    is_similar = False
    if iterations >= p["max_iterations"]:
        if not p["failure_after_max_iter"]:
            state.state = ITERATIONS
            return True
        state.state = FAILURE_AFTER_MAX_ITERATIONS
    cos, t2 = cos_t2(T_k, scalar, slip)
    trans_ok = t2 < p["trans_eps"] if "translation <" in slip else t2 <= p["trans_eps"]
    if cos >= state.rotation_threshold and trans_ok:
        if state.similar >= p["max_iterations_similar"]:
            state.state = TRANSFORM
            return True
        is_similar = True
    cur, prev = np.float64(mse), np.float64(state.prev_mse)
    with np.errstate(all="ignore"):
        d = abs(cur - prev)
        rel = d / prev
    fired = False
    abs_hit = d <= p["abs_mse"] if "abs <=" in slip else d < p["abs_mse"]
    if abs_hit:
        if state.similar >= p["max_iterations_similar"]:
            state.state, fired = ABS_MSE, True
        else:
            is_similar = True
    if not fired:
        rel_hit = rel <= p["rel_mse"] if "rel <=" in slip else rel < p["rel_mse"]
        if rel_hit:
            if state.similar >= p["max_iterations_similar"]:
                state.state, fired = REL_MSE, True
            else:
                is_similar = True
    if fired:
        if "prev_mse on the converging iteration" in slip:
            state.prev_mse = float(cur)
        return True
    if is_similar:
        state.similar += 1
    elif "similar count not reset" not in slip:
        state.similar = 0
    state.prev_mse = float(cur)
    return False


def compose(T_k, final, scalar, slip=()):
    """final = T_k * final in Scalar, Eigen's coefficient order, element-wise (not @, which reorders)."""
    S = np.float64 if (scalar == np.float64 or "composition in double" in slip) else np.float32
    a = np.asarray(T_k, dtype=np.float64).reshape(4, 4).astype(S)
    b = np.asarray(final, dtype=np.float64).reshape(4, 4).astype(S)
    if "final * T_k" in slip:
        a, b = b, a
    c = ((a[:, 0:1] * b[0:1, :] + a[:, 1:2] * b[1:2, :]) + a[:, 2:3] * b[2:3, :]) + a[:, 3:4] * b[3:4, :]
    return c.astype(scalar).astype(np.float64)


def start_align(state, p, slip=()):
    """icp.hpp:157-161 on the criteria object at the start of an align."""
    if p["rot_eps"] > 0:
        state.rotation_threshold = p["rot_eps"]
    if "prev_mse reset per align" in slip:
        state.prev_mse = DBL_MAX


def loop_reference(state, p, scalar, steps, final0=None, slip=()):
    """The do-while of icp.hpp:164-241 over recorded steps [(n_pairs, T_k, mse), ...] (T_k already in Scalar).
    Returns one record per executed pass: (state, converged, iterations, similar, prev_mse, final)."""
    start_align(state, p, slip)
    final = np.eye(4) if final0 is None else np.asarray(final0, dtype=np.float64).astype(scalar).astype(np.float64)
    iterations, out = 0, []
    for n_pairs, T_k, mse in steps:
        if n_pairs < 3:
            state.state = NO_CORRESPONDENCES
            out.append((NO_CORRESPONDENCES, False, iterations, state.similar, state.prev_mse, final.copy()))
            break
        final = compose(T_k, final, scalar, slip)
        iterations += 1
        converged = criteria_step(state, p, scalar, iterations, T_k, mse, slip)
        out.append((state.state, converged, iterations, state.similar, state.prev_mse, final.copy()))
        if state.state != NOT_CONVERGED:
            break
    return out


def pcl_mse(distances):
    """calculateMSE: the float distances summed in fp64 in list order, over double(n)."""
    d = np.asarray(distances, dtype=np.float32).astype(np.float64)
    return float(np.cumsum(d)[-1] / np.float64(d.size))


def same_bits(a, b):
    """bit for bit, except that any NaN equals any NaN (a NaN's sign and payload carry no meaning)"""
    a, b = np.asarray(a, dtype=np.float64).ravel(), np.asarray(b, dtype=np.float64).ravel()
    na, nb = np.isnan(a), np.isnan(b)
    return a.size == b.size and np.array_equal(na, nb) and a[~na].tobytes() == b[~nb].tobytes()


def stop_of(records):
    """(iterations, state, final bits) of a run's last record"""
    r = records[-1]
    return r[2], r[0], r[5].tobytes()


# ---------------------------------------------------------------------------------------------------------------------
# synthetic sequences
# ---------------------------------------------------------------------------------------------------------------------
def _rot(axis, ang):
    axis = np.asarray(axis, float) / np.linalg.norm(axis)
    K = np.array([[0, -axis[2], axis[1]], [axis[2], 0, -axis[0]], [-axis[1], axis[0], 0]])
    T = np.eye(4)
    T[:3, :3] = np.eye(3) + math.sin(ang) * K + (1 - math.cos(ang)) * K @ K
    return T


def _step_T(rng, scale, scalar):
    T = _rot(rng.normal(size=3), scale * rng.random() * 1e-2)
    T[:3, 3] = rng.normal(size=3) * scale * 1e-3
    return T.astype(scalar).astype(np.float64)


def _seq(rng, n, scalar, decay=0.5):
    """n steps whose motion shrinks geometrically and whose MSE lies on the dyadic grid k / 2^24 (exact differences)"""
    steps, mse, scale = [], rng.integers(2 ** 16, 2 ** 20), 1.0
    for _ in range(n):
        steps.append((1000, _step_T(rng, scale, scalar), float(mse) / 2 ** 24))
        scale *= decay * (0.5 + rng.random())
        mse = max(0, mse - int(rng.integers(0, max(1, mse // 3))))
    return steps


def _nb(x):
    """x and its neighbouring doubles"""
    return [math.nextafter(x, -math.inf), x, math.nextafter(x, math.inf)]


def _values(steps, scalar):
    """recorded values of a sequence a threshold can be set to: |dmse|, |dmse| / prev, cos and t^2 of each step"""
    out = dict(abs=[], rel=[], cos=[], t2=[])
    for k, (_, T, m) in enumerate(steps):
        c, t2 = cos_t2(T, scalar)
        out["cos"].append(c)
        out["t2"].append(t2)
        if k:
            prev = steps[k - 1][2]
            out["abs"].append(abs(m - prev))
            if prev > 0:
                out["rel"].append(abs(m - prev) / prev)
    return out


def float_double_split(rng, n=4000):
    """step transforms whose float and double cosines (or t^2) fall on opposite sides of a threshold between them"""
    found = []
    for _ in range(n):
        T = _step_T(rng, rng.random() * 0.1, np.float32)
        cf, tf = cos_t2(T, np.float32)
        cd, td = cos_t2(T, np.float32, slip=("cos, t^2 in double",))
        if cf != cd or tf != td:
            found.append((T, cf, cd, tf, td))
        if len(found) >= 12:
            break
    return found


def synthetic_cases(seed=20261019, n_random=20000):
    """[(label, scalar, params, steps, final0, prev_mse at the start, carried)]"""
    rng = np.random.default_rng(seed)
    cases = []
    # hand-made edges
    for scalar in (np.float32, np.float64):
        base = [(1000, np.eye(4), 0.5)]
        # |dmse| exactly at the absolute threshold and one ulp either side, the MSE values dyadic
        a = 2.0 ** -20
        for thr in _nb(a):
            cases.append(("abs at threshold", scalar, params(abs_mse=thr, trans_eps=-1.0, max_iterations=5),
                          base + [(1000, _step_T(rng, 1, scalar), 0.5 - a)] * 2, None, DBL_MAX, False))
        # |dmse| / prev exactly at the relative threshold and one ulp either side
        for thr in _nb(2.0 ** -20):
            cases.append(("rel at threshold", scalar, params(rel_mse=thr, abs_mse=0.0, trans_eps=-1.0, max_iterations=5),
                          base + [(1000, _step_T(rng, 1, scalar), 0.5 - 2.0 ** -21)] * 2, None, DBL_MAX, False))
        # prev = DBL_MAX, 0 and equal to cur; mse = 0
        for prev in (DBL_MAX, 0.0, 0.5):
            for m in (0.5, 0.0):
                for abs_thr, rel in ((1e-12, -DBL_MAX), (0.0, 1e-5), (0.0, 2.0), (1.0, -DBL_MAX)):
                    cases.append((f"prev {prev} mse {m}", scalar, params(abs_mse=abs_thr, rel_mse=rel, max_iterations=4),
                                  [(1000, _step_T(rng, 1, scalar), m)] * 3, None, prev, prev != DBL_MAX))
        # thresholds 0, negative, NaN; a relative threshold > 1 fires at iteration 1 against DBL_MAX
        for thr in (0.0, -1.0, math.nan, 1.5):
            cases.append((f"thresholds {thr}", scalar,
                          params(abs_mse=thr, rel_mse=thr, trans_eps=thr, rot_eps=thr, max_iterations=6),
                          _seq(rng, 6, scalar), None, DBL_MAX, False))
        # cos exactly at the rotation threshold, t^2 exactly at the translation threshold
        for _ in range(4):
            seq = _seq(rng, 5, scalar)
            v = _values(seq, scalar)
            k = int(rng.integers(0, 5))
            for thr in _nb(v["cos"][k]):
                cases.append(("cos at threshold", scalar, params(rot_eps=thr, trans_eps=1.0, abs_mse=0.0, max_iterations=8),
                              seq, None, DBL_MAX, False))
            for thr in _nb(v["t2"][k]):
                cases.append(("t2 at threshold", scalar, params(trans_eps=thr, rot_eps=-1.0, abs_mse=0.0, max_iterations=8),
                              seq, None, DBL_MAX, False))
                cases.append(("t2 at threshold, cos gate 0.5", scalar,
                              params(trans_eps=thr, rot_eps=0.5, abs_mse=0.0, max_iterations=8), seq, None, DBL_MAX, False))
        # max_iterations -1, 0, 1; max_iterations_similar 0..3; failure_after_max_iter on / off; a TRANSFORM that
        # fires on the iteration that also sets FAILURE_AFTER_MAX_ITERATIONS
        for mi in (-1, 0, 1, 3):
            for ms in range(4):
                for fail in (False, True):
                    seq = _seq(rng, 6, scalar, decay=0.1)
                    cases.append((f"max {mi} similar {ms} failure {fail}", scalar,
                                  params(max_iterations=mi, max_iterations_similar=ms, failure_after_max_iter=fail,
                                         trans_eps=1.0, rot_eps=0.5, abs_mse=0.0), seq, None, DBL_MAX, False))
        seq = [(1000, _step_T(rng, 100, scalar), 0.5), (1000, _step_T(rng, 100, scalar), 0.25),
               (1000, np.eye(4), 0.125)]
        for fail in (False, True):
            cases.append((f"TRANSFORM at max_iterations, failure {fail}", scalar,
                          params(max_iterations=3, failure_after_max_iter=fail, trans_eps=0.0, abs_mse=0.0), seq, None,
                          DBL_MAX, False))
        # NO_CORRESPONDENCES at iteration 1 and later
        cases.append(("no pairs at 1", scalar, params(), [(2, np.eye(4), 0.0)], None, DBL_MAX, False))
        cases.append(("no pairs at 3", scalar, params(abs_mse=0.0), _seq(rng, 2, scalar) + [(0, np.eye(4), 0.0)],
                      None, DBL_MAX, False))
    # float traces where the float and double evaluations fall on opposite sides of the threshold
    for T, cf, cd, tf, td in float_double_split(rng):
        seq = [(1000, T, 0.5), (1000, T, 0.25)]
        if cf != cd:
            thr = max(cf, cd)
            cases.append(("cos float / double split", np.float32, params(rot_eps=thr, trans_eps=1.0, abs_mse=0.0),
                          seq, None, DBL_MAX, False))
        if tf != td:
            thr = min(tf, td)
            cases.append(("t2 float / double split", np.float32, params(trans_eps=thr, rot_eps=-1.0, abs_mse=0.0),
                          seq, None, DBL_MAX, False))
    # seeded: thresholds at recorded values (and neighbours) of their own sequence, every knob drawn
    for i in range(n_random):
        scalar = np.float32 if i % 2 else np.float64
        seq = _seq(rng, int(rng.integers(1, 10)), scalar, decay=float(rng.choice([0.1, 0.5, 0.9])))
        if rng.random() < 0.05:
            k = int(rng.integers(0, len(seq)))
            seq[k] = (int(rng.integers(0, 3)), seq[k][1], seq[k][2])
        v = _values(seq, scalar)

        def pick(key, default):
            vals = v[key]
            if not vals or rng.random() < 0.3:
                return default
            return _nb(vals[int(rng.integers(0, len(vals)))])[int(rng.integers(0, 3))]
        p = params(max_iterations=int(rng.integers(-1, 11)), failure_after_max_iter=rng.random() < 0.3,
                   max_iterations_similar=int(rng.integers(0, 4)), rot_eps=pick("cos", 0.0),
                   trans_eps=pick("t2", 0.0), rel_mse=pick("rel", -DBL_MAX), abs_mse=pick("abs", 1e-12))
        carried = rng.random() < 0.2
        prev = float(rng.choice([m for _, _, m in seq])) if carried else DBL_MAX
        g = _step_T(rng, 100, scalar) if rng.random() < 0.3 else None
        cases.append(("seeded", scalar, p, seq, g, prev, carried))
    return cases


def run_reference(case, slip=()):
    label, scalar, p, steps, final0, prev, carried = case
    st = Criteria()
    st.prev_mse = prev
    return loop_reference(st, p, scalar, steps, final0, slip)


def _write_cases(path, cases):
    with open(path, "wb") as f:
        f.write(struct.pack("<i", len(cases)))
        for label, scalar, p, steps, final0, prev, carried in cases:
            f.write(struct.pack("<5i", int(scalar == np.float64), p["max_iterations"], int(p["failure_after_max_iter"]),
                                p["max_iterations_similar"], len(steps)))
            f.write(struct.pack("<5d", p["rot_eps"], p["trans_eps"], p["rel_mse"], p["abs_mse"], prev))
            g = np.eye(4) if final0 is None else np.asarray(final0, dtype=np.float64).astype(scalar).astype(np.float64)
            f.write(g.astype("<f8").tobytes())
            for n_pairs, T, m in steps:
                f.write(struct.pack("<id", int(n_pairs >= 3), m))
                f.write(np.asarray(T, dtype="<f8").tobytes())


def _read_records(path, n_cases):
    rec = np.dtype([("head", "<i4", 4), ("prev", "<f8"), ("final", "<f8", 16)])
    data, out, off = open(path, "rb").read(), [], 0
    for _ in range(n_cases):
        (n,) = struct.unpack_from("<i", data, off)
        off += 4
        out.append(np.frombuffer(data, rec, n, off))
        off += n * rec.itemsize
    assert off == len(data)
    return out


def _same(records, got):
    if len(records) != got.size:
        return False
    for r, g in zip(records, got):
        if (r[0], int(r[1]), r[2], r[3]) != tuple(int(x) for x in g["head"]):
            return False
        if not same_bits(r[4], g["prev"]) or not same_bits(r[5], g["final"]):
            return False
    return True


@pytest.fixture(scope="module")
def cases():
    return synthetic_cases()


@pytest.fixture(scope="module")
def host_records(cases, tmp_path_factory):
    from _sharded import host_program
    if shutil.which("g++") is None:
        pytest.skip("needs g++")
    d = tmp_path_factory.mktemp("loop")
    _write_cases(d / "in.bin", cases)
    out = host_program(d, "loop_host_test.cpp", args=(str(d / "in.bin"), str(d / "out.bin")), timeout=600)
    print(out.strip().splitlines()[0])
    return _read_records(d / "out.bin", len(cases))


def test_device_criteria_against_reference(cases, host_records):
    """has_converged_dev and mat4_mul_dev, compiled for the host, on every synthetic sequence: every step's state,
    converged flag, iteration count, similar count, previous-MSE bits and final bits equal the reference's."""
    bad = [(c[0], i) for i, (c, g) in enumerate(zip(cases, host_records)) if not _same(run_reference(c), g)]
    steps = sum(g.size for g in host_records)
    states = sorted({int(g["head"][-1, 0]) for g in host_records if g.size})
    print(f"\n{len(cases)} sequences, {steps} steps compared; final states seen: {states}")
    assert not bad, bad[:10]
    assert states == list(range(7))


def test_reference_rules_by_hand():
    """A few stops worked out from PCL's source by hand."""
    # a relative threshold > 1 fires at iteration 1 against DBL_MAX: |m - DBL_MAX| / DBL_MAX = 1 < 1.5
    T = _rot([0, 0, 1], 0.1)
    r = run_reference(("", np.float64, params(rel_mse=1.5, abs_mse=0.0), [(10, T, 0.5)], None, DBL_MAX, False))
    assert stop_of(r)[:2] == (1, REL_MSE) and r[-1][4] == DBL_MAX
    # equal MSE: |d| = 0 < 1e-12 fires ABS_MSE at iteration 2 and leaves prev at iteration 1's value
    r = run_reference(("", np.float64, params(), [(10, T, 0.5), (10, T, 0.5)], None, DBL_MAX, False))
    assert stop_of(r)[:2] == (2, ABS_MSE) and r[-1][4] == 0.5
    # a carried previous MSE equal to iteration 1's stops the second align at its iteration 1
    r = run_reference(("", np.float64, params(), [(10, T, 0.5), (10, T, 0.5)], None, 0.5, True))
    assert stop_of(r)[:2] == (1, ABS_MSE)
    # FAILURE_AFTER_MAX_ITERATIONS, then the identity: TRANSFORM on the same pass, converged
    r = run_reference(("", np.float64, params(max_iterations=1, failure_after_max_iter=True, abs_mse=0.0),
                       [(10, np.eye(4), 0.5)], None, DBL_MAX, False))
    assert stop_of(r)[:2] == (1, TRANSFORM) and r[-1][1]
    r = run_reference(("", np.float64, params(max_iterations=1, failure_after_max_iter=True, abs_mse=0.0),
                       [(10, T, 0.5)], None, DBL_MAX, False))
    assert stop_of(r)[:2] == (1, FAILURE_AFTER_MAX_ITERATIONS) and not r[-1][1]
    assert pcl_mse(np.float32([1e8, 1, -1e8])) == 1.0 / 3
    assert pcl_mse(np.float32([1, 2, 4])) == 7.0 / 3


# ---------------------------------------------------------------------------------------------------------------------
# the oracle's loop on recorded ICP runs
# ---------------------------------------------------------------------------------------------------------------------
def synthetic_pair_records(n=4000, seed=42):
    from test_gpu_parity import _synthetic_pair
    src, tgt = _synthetic_pair(np.random.default_rng(seed), n)
    return src, tgt, 0.05


def lattice_records():
    from test_rejectors_reference import lattice_pair
    tgt, src = lattice_pair()
    return src, tgt, 0.1


ORACLE_SCENES = {"synthetic pair": synthetic_pair_records, "lattice": lattice_records}
ESTIMATORS = {"svd": (0, False), "svd correlation": (0, True), "point-to-plane": (1, False), "symmetric": (2, False)}
OFF = dict(transformation_epsilon=-1.0, euclidean_fitness_epsilon=-DBL_MAX, mse_threshold_absolute=0.0)


def _recs(orc, pts):
    rec = np.zeros((pts.shape[0], 8), np.float32)
    rec[:, :3], rec[:, 3] = pts, 1
    nrm, _ = orc.Index(rec[:, :4]).normals_knn(rec[:, :4], 10, nthreads=os.cpu_count() or 8)
    rec[:, 4:7] = nrm[:, :3]
    return rec


_SCENES = {}


def oracle_scene(orc, name):
    if name not in _SCENES:
        src, tgt, gate = ORACLE_SCENES[name]()
        _SCENES[name] = (_recs(orc, src), _recs(orc, tgt), gate)
    return _SCENES[name]


def record_oracle(orc, src, tgt, gate, est, no_umeyama, dbl, K, guess=None, prev_mse=None):
    """Every iteration of a criteria-off run: max_iterations = k runs the same prefix and reports step k."""
    steps = []
    for k in range(1, K + 1):
        r = orc.icp_align_criteria(src, tgt, max_iterations=k, max_correspondence_distance=gate, estimator=est,
                                   svd_no_umeyama=no_umeyama, scalar_is_double=dbl, guess=guess, prev_mse=prev_mse,
                                   nthreads=os.cpu_count() or 8, **OFF)
        if r["state"] == NO_CORRESPONDENCES:
            steps.append((r["n_correspondences"], np.eye(4), 0.0))
            break
        assert r["iterations"] == k and r["state"] == ITERATIONS
        steps.append((r["n_correspondences"], r["last"], r["mse"]))
    return steps


def threshold_settings(steps, scalar):
    """each criterion alone at recorded values of the run (and the neighbouring doubles), plus mixed settings"""
    v = _values(steps, scalar)
    out = []
    for key, k in (("abs", "mse_threshold_absolute"), ("rel", "euclidean_fitness_epsilon")):
        for x in sorted(set(v[key]))[::2]:
            for t in _nb(x):
                out.append({**OFF, k: t})
    for x in sorted(set(v["t2"]))[::2]:
        for t in _nb(x):
            out.append({**OFF, "transformation_epsilon": t, "transformation_rotation_epsilon": -1.0})
    for x in sorted(set(v["cos"]))[::2]:
        if x > 0:
            for t in _nb(x):
                out.append({**OFF, "transformation_epsilon": 1.0, "transformation_rotation_epsilon": t})
    for ms in (1, 2, 3):
        if v["abs"]:
            out.append({**OFF, "mse_threshold_absolute": float(np.quantile(v["abs"], 0.5)),
                        "max_iterations_similar_transforms": ms})
    return out


def _oracle_params(kw, K):
    return params(max_iterations=K, failure_after_max_iter=kw.get("failure_after_max_iter", False),
                  max_iterations_similar=kw.get("max_iterations_similar_transforms", 0),
                  rot_eps=kw.get("transformation_rotation_epsilon", 0.0), trans_eps=kw["transformation_epsilon"],
                  rel_mse=kw["euclidean_fitness_epsilon"], abs_mse=kw["mse_threshold_absolute"])


RECORDED = {}   # (scene, estimator, scalar) -> steps, for the teeth


# the lattice's k-NN normals are all one plane, so the normal equations of the two normal-based objectives are singular
ORACLE_RUNS = [(s, e) for s in ORACLE_SCENES for e in ESTIMATORS if s != "lattice" or e.startswith("svd")]


@pytest.mark.parametrize("dbl", [False, True], ids=["float", "double"])
@pytest.mark.parametrize("scene,est", ORACLE_RUNS)
def test_oracle_against_reference(orc, scene, est, dbl):
    """The oracle's loop, with every threshold at a recorded value of its own criteria-off run and at the neighbouring
    doubles, stops where loop_reference says: iterations, state, converged and final bits.  A second align of the same
    criteria object from the first one's result carries the previous MSE."""
    src, tgt, gate = oracle_scene(orc, scene)
    e, no_u = ESTIMATORS[est]
    scalar = np.float64 if dbl else np.float32
    K = 8
    steps = record_oracle(orc, src, tgt, gate, e, no_u, dbl, K)
    RECORDED[(scene, est, dbl)] = steps
    settings = threshold_settings(steps, scalar)
    stops = set()
    for kw in settings:
        r = orc.icp_align_criteria(src, tgt, max_iterations=K, max_correspondence_distance=gate, estimator=e,
                                   svd_no_umeyama=no_u, scalar_is_double=dbl, nthreads=os.cpu_count() or 8,
                                   **{k: v for k, v in kw.items() if k != "max_iterations_similar_transforms"},
                                   max_iterations_similar_transforms=kw.get("max_iterations_similar_transforms", 0))
        want = loop_reference(Criteria(), _oracle_params(kw, K), scalar, steps)
        assert (r["iterations"], r["state"], r["converged"]) == (want[-1][2], want[-1][0], want[-1][1]), (kw, r, want[-1][:4])
        assert same_bits(r["final"], want[-1][5]), kw
        assert same_bits(r["prev_mse"], want[-1][4]), kw
        stops.add((r["iterations"], r["state"]))
    print(f"\n{scene}, {est}, {'double' if dbl else 'float'}: {len(settings)} settings, stops {sorted(stops)}")
    assert len(stops) >= 3
    # across aligns: the same criteria object aligns again from its own result
    kw = {**OFF, "mse_threshold_absolute": 1.0}
    first = orc.icp_align_criteria(src, tgt, max_iterations=K, max_correspondence_distance=gate, estimator=e,
                                   svd_no_umeyama=no_u, scalar_is_double=dbl, nthreads=os.cpu_count() or 8, **kw)
    steps2 = record_oracle(orc, src, tgt, gate, e, no_u, dbl, 3, guess=first["final"])
    second = orc.icp_align_criteria(src, tgt, max_iterations=K, max_correspondence_distance=gate, estimator=e,
                                    svd_no_umeyama=no_u, scalar_is_double=dbl, guess=first["final"],
                                    prev_mse=first["prev_mse"], nthreads=os.cpu_count() or 8, **kw)
    st = Criteria()
    st.prev_mse = first["prev_mse"]
    want = loop_reference(st, _oracle_params(kw, K), scalar, steps2, final0=first["final"])
    assert (second["iterations"], second["state"]) == stop_of(want)[:2] == (1, ABS_MSE)
    assert same_bits(second["final"], want[-1][5])
    fresh = loop_reference(Criteria(), _oracle_params(kw, K), scalar, steps2, final0=first["final"])
    assert stop_of(fresh)[:2] == (2, ABS_MSE)


def test_teeth(cases):
    """Each slip of the rules changes at least one predicted stop (iterations or state; final bits for the two
    composition slips) on the synthetic set (single aligns, and pairs of aligns of one criteria object) or on the
    oracle's recorded runs."""
    rows = []
    for slip in SLIPS:
        changed = 0
        for c in cases:
            a, b = run_reference(c), run_reference(c, slip=(slip,))
            key = (lambda s: s) if slip in ("final * T_k", "composition in double") else (lambda s: s[:2])
            changed += key(stop_of(a)) != key(stop_of(b))
        # two aligns of one criteria object: consecutive sequences of the set, under the first one's settings
        for c1, c2 in zip(cases[::2], cases[1::2]):
            if c1[1] != c2[1]:
                continue
            a, b = Criteria(), Criteria()
            loop_reference(a, c1[2], c1[1], c1[3], c1[4])
            loop_reference(b, c1[2], c1[1], c1[3], c1[4], slip=(slip,))
            ra = loop_reference(a, c1[2], c1[1], c2[3], c2[4])
            rb = loop_reference(b, c1[2], c1[1], c2[3], c2[4], slip=(slip,))
            key = (lambda s: s) if slip in ("final * T_k", "composition in double") else (lambda s: s[:2])
            changed += key(stop_of(ra)) != key(stop_of(rb))
        rec = 0
        for (scene, est, dbl), steps in RECORDED.items():
            scalar = np.float64 if dbl else np.float32
            for kw in threshold_settings(steps, scalar):
                p = _oracle_params(kw, 8)
                a = loop_reference(Criteria(), p, scalar, steps)
                b = loop_reference(Criteria(), p, scalar, steps, slip=(slip,))
                key = (lambda s: s) if slip in ("final * T_k", "composition in double") else (lambda s: s[:2])
                rec += key(stop_of(a)) != key(stop_of(b))
        rows.append((slip, changed, rec))
    print(f"\n{'slip':40s} {'synthetic':>10s} {'recorded':>9s}")
    for slip, c, r in rows:
        print(f"{slip:40s} {c:10d} {r:9d}")
    assert all(c + r > 0 for _, c, r in rows), rows
