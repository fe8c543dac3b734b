"""The exchange of a target map sharded across ranks (pcl_b200/csrc/shard_target_kernels.cuh, driven by icp.cu:
exchange_shard_matches and fitness_score_sharded), compiled for the host: no GPU needed."""
import _sharded as S


@S.needs_host_compiler
def test_sharded_target_table_sets_on_the_host(tmp_path):
    """1 / 2 / 3 / 5 / 8 simulated ranks, both exchange protocols: the gathered match and record of every query equal the
    brute-force (d2, id) argmin over the whole map — exact ties across ranks, ids near 2^31 - 1, a rank out of reach, a
    random partition, points held by two ranks — and the fitness reduction, reading the keys through peer_table_set, counts exactly."""
    out = S.host_program(tmp_path, "shard_target_host_test.cpp", timeout=900)
    assert any(l.startswith("a tile out of reach") and "R=8 nccl" in l for l in out.splitlines())
    assert "DIFFERS" not in out
