"""Every device correspondence rejector against the reference of tests/test_rejectors_reference.py, bit for bit:
stand-alone through pclb200_reject (host and device arrays), and inside the ICP loop, where every iteration's list
after the chain must equal the reference chain applied to the reference 1-NN (or normal-shooting) list of the source
the device moved.  Which settings a loop ran with is recorded per path, and every path must have been served by one of
the far scenes.  Needs an H100: run with -m gpu."""
import ctypes as C
import math
import os
import sys
import time
from collections import defaultdict

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_consumers_reference as CR  # noqa: E402
import test_rejectors_reference as RR  # noqa: E402
import test_search_reference as R  # noqa: E402
from test_gpu_search_reference import _icp_pair  # noqa: E402
from test_normals_reference import knn_sets  # noqa: E402

pytestmark = pytest.mark.gpu

FAR_SCENES = ("map_1e5", "object_far_out", "straddle")
LOOP_SCENES = FAR_SCENES + ("lattice",)
SERVED = defaultdict(set)   # path -> scenes that went through it
STEPS = defaultdict(int)    # path -> loop iterations compared
T0 = [0.0]


@pytest.fixture(scope="module")
def gpu():
    import pcl_b200
    pcl_b200.lib()
    ctx = pcl_b200.Context(0)
    T0[0] = time.time()
    yield pcl_b200, ctx
    ctx.close()
    print(f"\n{'path':48s} {'steps':>6s}  scenes")
    for path in sorted(SERVED):
        print(f"{path:48s} {STEPS[path]:6d}  {', '.join(sorted(SERVED[path]))}")
    print(f"test_gpu_rejectors_reference.py: {time.time() - T0[0]:.1f} s")


def _served(path, scene, steps=1):
    SERVED[path].add(scene)
    STEPS[path] += steps


def _reject_c(P, ctx, c, kind, p, mn, to_device_in, to_device_out):
    """pclb200_reject straight through the C entry point, the input and / or the output in torch device memory."""
    import torch
    r = P.Rejector(kind, mn, float(p))
    src = np.ascontiguousarray(c, dtype=P.CORR_DTYPE)
    n = src.size
    if to_device_in:
        tin = torch.from_numpy(src.view(np.int32).reshape(n, 3).copy()).cuda()
        pin = C.c_void_p(tin.data_ptr())
    else:
        pin = C.c_void_p(src.ctypes.data)
    if to_device_out:
        tout = torch.zeros((max(n, 1), 3), dtype=torch.int32, device="cuda")
        pout = C.c_void_p(tout.data_ptr())
    else:
        hout = np.zeros(max(n, 1), P.CORR_DTYPE)
        pout = C.c_void_p(hout.ctypes.data)
    m, med = C.c_size_t(), C.c_double()
    rc = P.lib().pclb200_reject(ctx.h, C.byref(r), pin, n, pout, C.byref(m), C.byref(med))
    assert rc == 0, rc
    if to_device_out:
        torch.cuda.synchronize()
        out = tout.cpu().numpy().reshape(-1).view(P.CORR_DTYPE)[:m.value].copy()
    else:
        out = hout[:m.value].copy()
    return out, float(med.value)


# ---------------------------------------------------------------------------------------------------------------------
# stand-alone
# ---------------------------------------------------------------------------------------------------------------------
def test_standalone_synthetic(gpu):
    """Every synthetic list and parameter of the CPU file: records, order and median bit for bit."""
    P, ctx = gpu
    RR.check_standalone(lambda c, k, p, m: ctx.reject(c, k, p=p, min_correspondences=m), RR.SYNTH)


@pytest.mark.parametrize("name", list(R.SCENES))
def test_standalone_scene_lists(gpu, name):
    P, ctx = gpu
    lists = RR.scene_lists(name)
    RR.check_standalone(lambda c, k, p, m: ctx.reject(c, k, p=p, min_correspondences=m), lists)


def test_standalone_device_arrays(gpu):
    """The C entry point with the input, the output or both in device memory (torch), on lists with every special
    distance and on a scene list."""
    P, ctx = gpu
    lists = {k: v for k, v in RR.SYNTH.items() if k.startswith(("n=257 ", "n=4097 ", "n=1 "))}
    lists.update({k: v for k, v in RR.scene_lists("map_1e5").items() if "ungated" in k or "subset" in k})
    for din, dout in ((True, True), (True, False), (False, True)):
        RR.check_standalone(lambda c, k, p, m: _reject_c(P, ctx, c, k, p, m, din, dout), lists)


def test_standalone_count_past_float_precision(gpu):
    """2^24 + 5 entries at overlap 1.0: float(n) rounds to 2^24 + 4, so PCL's count trims the farthest entry; the
    median of the same list."""
    P, ctx = gpu
    n = 2 ** 24 + 5
    rng = np.random.default_rng(71)
    c = RR.corr(np.arange(n, dtype=np.int32), rng.integers(0, n // 3, n).astype(np.int32),
                np.round(rng.random(n, dtype=np.float32) * 4096) / np.float32(4096))
    assert RR.trimmed_keep(1.0, n, 0) == n - 1
    for kind, p in ((RR.TRIMMED, 1.0), (RR.MEDIAN, 1.0)):
        got, gmed = ctx.reject(c, kind, p=p)
        want, wmed = RR.reject_ref(c, kind, p)
        assert got.size == want.size and got.tobytes() == want.tobytes(), (kind, got.size, want.size)
        assert gmed == wmed, (kind, gmed, wmed)


# ---------------------------------------------------------------------------------------------------------------------
# inside the ICP loop
# ---------------------------------------------------------------------------------------------------------------------
def lattice_icp_pair():
    """The lattice pair of the CPU file (exact ties everywhere in the first iteration) and its gate."""
    tgt, src = RR.lattice_pair()
    return tgt, src, 0.1


SCENE_CACHE = {}


def loop_scene(name, orc):
    """(target records, source records, gate): 8 floats per point, xyz 1 | normal (the oracle's k = 10 normals) 0;
    every 97th source row NaN (for the is_dense = 0 cases)."""
    if name not in SCENE_CACHE:
        SCENE_CACHE.clear()
        tgt, src, gate = lattice_icp_pair() if name == "lattice" else _icp_pair(name)
        recs = []
        for pts in (tgt, src):
            rec = np.zeros((pts.shape[0], 8), np.float32)
            rec[:, :3], rec[:, 3] = pts, 1
            nrm, _ = orc.Index(rec[:, :4]).normals_knn(rec[:, :4], 10, nthreads=os.cpu_count() or 8)
            rec[:, 4:7] = nrm[:, :3]
            recs.append(rec)
        SCENE_CACHE[name] = (recs[0], recs[1], gate)
    return SCENE_CACHE[name]


CHAIN4 = RR.CHAIN4
# name -> (chain, loop settings); settings: est (svd / p2p), dbl, track (on / off / auto), corr (nearest /
# reciprocal / normal_shooting), subset, nan_rows
CASES = {
    "distance": ([(RR.DISTANCE, None, 0)], dict(track="on")),
    "median": ([(RR.MEDIAN, 1.5, 0)], dict(track="off", dbl=True)),
    "one-to-one": ([(RR.ONE_TO_ONE, 0.0, 0)], dict(track="auto")),
    "trimmed": ([(RR.TRIMMED, 0.8, 0)], dict(est="p2p")),
    "one-to-one, trimmed": ([(RR.ONE_TO_ONE, 0.0, 0), (RR.TRIMMED, 0.6, 0)], dict(track="on")),
    "trimmed, one-to-one": ([(RR.TRIMMED, 0.6, 0), (RR.ONE_TO_ONE, 0.0, 0)], dict(track="off", dbl=True)),
    "chain of four, reciprocal": (CHAIN4, dict(corr="reciprocal", dbl=True)),
    "chain of four, subset, NaN rows": (CHAIN4, dict(subset=True, nan_rows=True, track="auto")),
    "surface normal + chain of four": ([(RR.SURFACE_NORMAL, 0.7, 0)] + CHAIN4, dict(est="p2p")),
    "normal shooting + chain of four": (CHAIN4, dict(corr="normal_shooting")),
    "fewer than 3 pairs": ([(RR.ONE_TO_ONE, 0.0, 0), (RR.TRIMMED, 0.0, 2)], dict()),
}


def _chain_for(chain, gate):
    """DISTANCE with p = None takes half the gate."""
    return [(k, 0.5 * gate if p is None else p, m) for k, p, m in chain]


def run_loop_case(P, ctx, orc, name, case):
    chain0, cfg = CASES[case]
    tgt, src, gate = loop_scene(name, orc)
    chain = _chain_for(chain0, gate)
    est, dbl = cfg.get("est", "svd"), cfg.get("dbl", False)
    corr = cfg.get("corr", "nearest")
    track = {"on": P.TRACK_ON, "off": P.TRACK_OFF, "auto": P.TRACK_AUTO}[cfg.get("track", "auto")]
    src = src.copy()
    if cfg.get("nan_rows"):
        src[::97, :3] = np.nan
    nt = est == "p2p" or corr == "normal_shooting" or any(k == RR.SURFACE_NORMAL for k, _, _ in chain)
    ind = np.random.default_rng(37).permutation(src.shape[0])[: (2 * src.shape[0]) // 3].astype(np.int32) \
        if cfg.get("subset") else None
    kind = P.CORR_NORMAL_SHOOTING if corr == "normal_shooting" else 0
    gate_kw = {} if kind else dict(max_correspondence_distance=gate)  # normal shooting runs ungated
    s = P.Icp(ctx, max_iterations=6, estimator=P.EST_POINT_TO_PLANE_LLS if est == "p2p" else P.EST_SVD,
              scalar_is_double=int(dbl), use_reciprocal=int(corr == "reciprocal"), with_normals_transform=int(nt),
              correspondence_kind=kind, correspondence_k=10, is_dense=0 if cfg.get("nan_rows") else 1,
              track_mode=track, transformation_epsilon=0.0, euclidean_fitness_epsilon=-1.0,
              mse_threshold_absolute=0.0, **gate_kw)
    T4 = np.ascontiguousarray(tgt[:, :4])
    tidx = P.Index(ctx, T4)
    s.set_target(tidx, normals=np.ascontiguousarray(tgt[:, 4:8]))
    s.set_rejectors(chain)
    s.set_source(np.ascontiguousarray(src[:, :4]), normals=np.ascontiguousarray(src[:, 4:8]) if nt else None,
                 indices=ind)
    cur = src.copy()
    normals = (None, np.ascontiguousarray(tgt[:, 4:7]))
    label = f"{case} [{est}, {'double' if dbl else 'float'}, tracking {cfg.get('track', 'auto')}, {corr}]"
    for it in range(6):
        st = s.iterate(1)
        got = s.get_correspondences()
        if kind:
            k = 10
            ki, kd = knn_sets(T4, cur[:, :4], k, return_d2=True)
            base = CR.normals_corr_ref(kind, cur[:, :4], cur[:, 4:7], T4, tgt[:, 4:7], ki, kd, k, indices=ind)
        else:
            ri, rd = knn_sets(T4, cur[:, :4], 1, return_d2=True)
            back = R.reciprocal_back(cur[:, :4], T4) if corr == "reciprocal" else None
            base = R.corr_ref(ri[:, 0], rd[:, 0], gate, indices=ind, back=back)
        want = RR.chain_ref(base, chain, normals=(np.ascontiguousarray(cur[:, 4:7]), normals[1]))
        assert got.size == want.size and got.tobytes() == want.tobytes(), \
            (name, label, it, got.size, want.size, base.size)
        assert st["n_correspondences"] == want.size, (name, label, it, st["n_correspondences"], want.size)
        _served(label.split(" [")[0], name)
        for path in (f"estimator {est}", f"scalar {'double' if dbl else 'float'}", f"tracking {cfg.get('track', 'auto')}",
                     f"correspondences {corr}") + (("index subset",) if ind is not None else ()) + \
                (("is_dense = 0, NaN rows",) if cfg.get("nan_rows") else ()):
            _served(path, name)
        if st["state"] == 5:  # NO_CORRESPONDENCES: the list that made the loop stop
            assert want.size < 3, (name, label, it, want.size)
            _served("NO_CORRESPONDENCES", name)
            return
        assert st["iterations"] == it + 1 and want.size >= 3, (name, label, it, st)
        d = want["distance"].astype(np.float64)
        assert abs(st["mse"] - math.fsum(d) / d.size) <= 1e-15 * abs(st["mse"]), (name, label, it, st["mse"])
        cur = orc.transform(cur, st["last"], scalar_is_double=dbl, mode=1 if nt else 0, normal_off=4 if nt else -1)
        if st["state"] != 0:
            return
    assert case != "fewer than 3 pairs", (name, "the loop did not stop")


@pytest.mark.parametrize("case", list(CASES))
@pytest.mark.parametrize("name", LOOP_SCENES)
def test_loop_chain_every_iteration(gpu, orc, name, case):
    """Up to 6 single steps; each step's list after the chain equals the reference chain on the reference list of
    the source rebuilt from the device's increments, in source-position order; n_correspondences and mse follow it."""
    P, ctx = gpu
    run_loop_case(P, ctx, orc, name, case)


def test_every_path_was_served_by_a_far_scene(gpu):
    """Each chain and each loop setting went through at least one far scene (run after them; skipped when they
    were deselected)."""
    if not all(any(name in v for v in SERVED.values()) for name in LOOP_SCENES):
        pytest.skip("needs every loop test of this file in the same run")
    for path in list(CASES) + ["estimator svd", "estimator p2p", "scalar float", "scalar double", "tracking on",
                               "tracking off", "tracking auto", "correspondences nearest", "correspondences reciprocal",
                               "correspondences normal_shooting", "index subset", "is_dense = 0, NaN rows",
                               "NO_CORRESPONDENCES"]:
        assert SERVED[path] & set(FAR_SCENES), (path, SERVED[path])
