"""The correspondence lists of a sharded map (pcl_b200/csrc/shard_target_kernels.cuh: k_tile_keys, k_keys_to_corr, and
k_knn_keys, k_merge_rows, k_candidate_scores, k_select_sharded; driven by icp.cu: correspondences_sharded,
correspondences_normals_sharded), compiled for the host: no GPU needed."""
import _sharded as S


@S.needs_host_compiler
def test_sharded_corr_lists_on_the_host(tmp_path):
    """1 / 2 / 3 / 5 / 8 simulated ranks, both exchange protocols, nearest and reciprocal, three gates and a descending
    subset: every rank's list equals the brute-force list over the whole map byte for byte — exact ties across ranks, ids
    held by two ranks, ids near 2^31 - 1, a tile out of reach, non-finite and repeated source points.  Normal shooting and
    back projection, k = 1 / 10 / 40, two gates: every rank's list equals select_by_normals over the whole map's k nearest,
    with NaN normals, tiles smaller than k and a whole map smaller than k."""
    out = S.host_program(tmp_path, "shard_corr_host_test.cpp", timeout=900)
    assert any(l.startswith("a tile out of reach") and "R=8 nccl  reciprocal" in l for l in out.splitlines())
    assert any(l.startswith("normals, small map") and "R=8 nccl" in l and "k=40 keff=35" in l for l in out.splitlines())
    assert "DIFFERS" not in out
