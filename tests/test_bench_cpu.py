"""bench.py's roofline denominators are the figures of SURVEY.md §8(d), and its helpers behave."""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402


def test_algorithmic_work_matches_the_survey_figures():
    a = bench.algorithmic(bench.LLAMA3_8B, 32, 1024, 128)
    assert abs(a["layer_params"] - 218_112_000) <= 2 * 4096                # the survey also counts the two norm vectors
    assert abs(a["weight_bytes"] - 15.01e9) < 0.01e9                    # 32 layers + lm_head, bf16
    assert a["kv_bytes_per_token"] == 131_072
    assert abs(a["decode_bytes_per_step"] - 19.57e9) < 0.01e9          # -> 5.84 ms at 3.35 TB/s
    assert abs(a["prefill_flops"] - 466e12) < 1e12                      # 457.4 GEMM + 8.8 causal attention + lm_head
    half = bench.algorithmic(bench.LLAMA3_8B, 32, 1024, 128, tp=2)
    assert abs(half["decode_bytes_per_step"] * 2 - a["decode_bytes_per_step"]) < 1 and abs(half["prefill_flops"] * 2 - a["prefill_flops"]) < 1
    m = bench.algorithmic(bench.MIXTRAL_8X7B, 32, 1024, 128, tp=4)
    assert abs(m["weight_bytes"] * 4 - 93.4e9) < 0.5e9                  # all 8 experts stream (46.7 B params incl. the embedding)


def test_cpu_thread_policy_and_peaks():
    n = bench.usable_cores()
    assert 1 <= n <= (os.cpu_count() or 1)
    p = bench.load_peaks()
    assert p["hbm_gbs"] > 1000 and p["tf_sustained"] <= p["tf_burst"]
    assert json.dumps(p)


def test_both_arms_share_one_config_dict():
    """VERDICT r01: the reference arm mislabelled its workload and `same_config` was false.  Both arms now build `config`
    from one function of (model, batch, prompt, gen, gpus), and it states what one reference step is."""
    a = bench.workload_config("Llama-3-8B", 32, 1024, 128, 4)
    assert a == bench.workload_config("Llama-3-8B", 32, 1024, 128, 4)
    assert a["global_batch"] == 32 and a["parallelism"] == "tp4" and "batch 1 x 1024-in/128-out in full" in a["reference_sample"]
    src = open(bench.__file__).read()
    assert src.count('"config": workload_config(') == 2          # the GPU arm and the reference arm, nothing hand-written
