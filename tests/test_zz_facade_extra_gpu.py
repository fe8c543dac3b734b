"""Second facade test program (pcl_b200/pcl_compat/tests/test_facade_extra.cpp): the pcl::search::Search overloads,
CorrespondenceEstimation::setPointRepresentation[Reciprocal], the DefaultConvergenceCriteria thresholds, the sample-consensus
rejector (the reference's golden 97 pairs) and the reference's ICP-with-rejectors test — facade surface added after the main
facade program's last run on hardware; the same program passes on the CPU against the oracle-backed test double
(tests/test_facade_on_oracle.py).  Named to run last."""
import os
import subprocess

import pytest

from test_facade_gpu import FACADE, _write_ascii_pcd, _write_binary_pcd, _write_golden


@pytest.mark.gpu
def test_facade_extra_api(golden, tmp_path):
    subprocess.check_call(["make", "-C", FACADE, "-s", "tests/test_facade_extra"])
    _write_ascii_pcd(tmp_path / "bun0.pcd", golden["bun0"])
    _write_binary_pcd(tmp_path / "bun4.pcd", golden["bun4"])
    _write_golden(tmp_path / "golden.txt", golden)
    r = subprocess.run([os.path.join(FACADE, "tests", "test_facade_extra"), str(tmp_path / "bun0.pcd"),
                        str(tmp_path / "bun4.pcd"), str(tmp_path / "golden.txt")], capture_output=True, text=True)
    print(r.stdout[-3000:], r.stderr[-2000:])
    assert r.returncode == 0, r.stdout[-3000:]
    assert "PASSED" in r.stdout


@pytest.mark.gpu
def test_facade_criteria_carry_over(golden, tmp_path):
    """pcl_b200/pcl_compat/tests/test_facade_loop.cpp on the device: a second align() of one IterativeClosestPoint
    compares its first iteration with the previous MSE the first align recorded, on the fused device loop and on the
    staged loop."""
    subprocess.check_call(["make", "-C", FACADE, "-s", "tests/test_facade_loop"])
    _write_ascii_pcd(tmp_path / "bun0.pcd", golden["bun0"])
    _write_binary_pcd(tmp_path / "bun4.pcd", golden["bun4"])
    r = subprocess.run([os.path.join(FACADE, "tests", "test_facade_loop"), str(tmp_path / "bun0.pcd"),
                        str(tmp_path / "bun4.pcd")], capture_output=True, text=True)
    print(r.stdout[-3000:], r.stderr[-2000:])
    assert r.returncode == 0 and "PASSED" in r.stdout, r.stdout[-3000:]


@pytest.mark.gpu
def test_icp_command_line_example(golden, tmp_path):
    """pcl_b200/pcl_compat/examples/iterative_closest_point.cpp — the flow of the reference's tools/iterative_closest_point.cpp
    (blob PCD in, PointNormal ICP<double> with injected estimators and a one-to-one rejector, concatenateFields, blob PCD
    out) end to end on the device."""
    import numpy as np
    subprocess.check_call(["make", "-C", FACADE, "-s", "examples/iterative_closest_point"])
    _write_binary_pcd(tmp_path / "bun0.pcd", golden["bun0"])
    _write_ascii_pcd(tmp_path / "bun4.pcd", golden["bun4"])
    out = tmp_path / "aligned.pcd"
    r = subprocess.run([os.path.join(FACADE, "examples", "iterative_closest_point"), str(tmp_path / "bun0.pcd"),
                        str(tmp_path / "bun4.pcd"), str(out), "50", "0.05"], capture_output=True, text=True)
    print(r.stdout[-3000:], r.stderr[-2000:])
    assert r.returncode in (0, 1), r.stdout[-2000:]          # 1 = ran, not converged
    assert "has converged" in r.stdout
    text = out.read_text().splitlines()
    hdr = {ln.split()[0]: ln.split()[1:] for ln in text[:11] if ln and not ln.startswith("#")}
    assert hdr["FIELDS"][:3] == ["x", "y", "z"] and "normal_x" in hdr["FIELDS"] and hdr["POINTS"] == ["397"]
    body = np.array([[float(t) for t in ln.split()] for ln in text[11:] if ln.strip()])
    assert body.shape[0] == 397 and np.isfinite(body[:, :3]).all()
    # the aligned cloud is closer to the target than the input was (mean nearest-neighbour distance, brute force)
    tgt = np.asarray(golden["bun4"], dtype=np.float64)[:, :3]
    def mean_nn(a):
        return np.sqrt(((a[:, None, :] - tgt[None, :, :]) ** 2).sum(-1).min(1)).mean()
    assert mean_nn(body[:, :3]) < mean_nn(np.asarray(golden["bun0"], dtype=np.float64)[:, :3])


@pytest.mark.gpu
def test_host_register_pinned_buffers(orc):
    """pclb200_host_register / _unregister (the pinned-reader half of SURVEY.md §8f #3): a page-locked caller buffer gives the
    same align as a pageable one; registering twice, unregistering an unknown buffer and registering a device pointer are
    refused with PCLB200_ERR_INVALID."""
    import numpy as np
    import pcl_b200 as P
    ctx = P.Context(0)
    rng = np.random.default_rng(5)
    tgt = P.xyz1(rng.random((200_000, 3), dtype=np.float32))
    a = np.deg2rad(2.0)
    R = np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]])
    src = P.xyz1((tgt[:, :3].astype(np.float64) @ R.T + [0.004, -0.003, 0.002]).astype(np.float32))
    idx = P.Index(ctx, tgt)
    kw = dict(max_iterations=20, max_correspondence_distance=0.05)
    plain = P.icp_align(ctx, src.copy(), idx, **kw)
    ctx.host_register(src)
    try:
        pinned = P.icp_align(ctx, src, idx, **kw)
        with pytest.raises(P.Pclb200Error) as e:
            ctx.host_register(src)
        assert e.value.code == P.ERR_INVALID
    finally:
        ctx.host_unregister(src)
    assert np.array_equal(plain["final"], pinned["final"]) and plain["iterations"] == pinned["iterations"]
    with pytest.raises(P.Pclb200Error) as e:
        ctx.host_unregister(src)
    assert e.value.code == P.ERR_INVALID
    ctx.close()
