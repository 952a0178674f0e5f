"""bench.py: the arithmetic behind the reported roofline (CPU only; the timed legs need an H100)."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402


def test_algorithmic_bytes_match_survey_8d():
    """SURVEY.md 8(d): packed index bytes + x + y per launch.  Llama-3-8B, b = 24: 2,622,488,576 B per token
    (the figure the round-1 review recomputed), 20,488,192 B per launch at 128 fused launches."""
    m, q, metric, cfg = bench.MODELS["llama3-8b"]
    tot = bench.algorithmic_bytes(m, q)
    assert tot == 2_622_488_576
    assert tot // 128 == 20_488_192
    # one 4096 x 4096 linear: 512 index rows x 3072 words + x + y
    assert 512 * 3072 * 4 + 4096 * 2 + 4096 * 2 == 6_307_840
    # tensor-parallel shards: index bytes split, x replicated
    for world in (2, 4, 8):
        part = bench.algorithmic_bytes(m, q, world=world)
        assert tot / world < part < tot / world + 32 * 7 * 2 * 14336


def test_models_are_the_baseline_configs():
    base = json.load(open(os.path.join(ROOT, "BASELINE.json")))
    m8, q8, metric8, cfg8 = bench.MODELS["llama3-8b"]
    assert (m8["layers"], m8["hidden"], m8["kv"], m8["ffn"]) == (32, 4096, 1024, 14336)
    assert (q8["vector_len"], q8["num_centroids"], q8["num_res_centroids"]) == (8, 65536, 256)
    m70, q70, _, _ = bench.MODELS["llama3-70b"]
    assert (m70["layers"], m70["hidden"], m70["kv"], m70["ffn"]) == (80, 8192, 1024, 28672)
    assert base["metric"].startswith("decode tokens/sec Llama-3-8B 2-bit") and metric8.startswith("decode tokens/sec Llama-3-8B 2-bit")
    s = bench.workload_string(m8, q8, cfg8)
    assert "224 VPTQ linears" in s and "(b=24)" in s

