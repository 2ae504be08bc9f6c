"""bench.py output contract (CPU side): the reference arm prints ONE JSON line with the keys the driver reads, and the
flop / metric bookkeeping of the GPU arm matches the analytic FLOP counts."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_reference_arm_prints_one_json_line_with_the_contract_keys():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--steps", "1",
                        "--warmup", "0", "--cpu-batch", "1", "--no-matrix"], capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [ln for ln in r.stdout.splitlines() if ln.strip()]
    assert len(lines) == 1, r.stdout
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["higher_is_better"] is True and d["unit"] == "images/sec"
    assert d["metric"].startswith("images/sec ViT-B/16") and d["n_gpus"] == 1 and d["steps"] == 1
    assert d["value"] > 0 and d["ms_per_step"] > 0 and d["vs_baseline"] is None
    cb = d["cpu_baseline"]
    # the unmodified reference from baseline/_ref when it is installed (kind "reference"), else the oracle port
    installed = os.path.isdir(os.path.join(ROOT, "baseline", "_ref", "vit_pytorch"))
    assert cb["kind"] == ("reference" if installed else "port") and cb["cores"] == os.cpu_count()
    assert cb["value"] == d["value"] and ("baseline/_ref" in cb["sample"] or "oracle" in cb["sample"])
    assert d["dtype"] == "bf16" and d["config"]["threads"] == os.cpu_count() and d["config"]["cpu"]
    e = d["e2e"]
    assert e["value"] == d["value"] and e["h2d_bytes_per_step"] == 0 and e["d2h_bytes_per_step"] == 0
    assert "workload" in d["config"] and "model" not in d["config"]


def test_algorithmic_flops_match_the_survey():
    sys.path.insert(0, ROOT)
    import bench
    from oracle import vit_oracle as O
    assert abs(O.flops_per_image(**bench.VIT_B16) / 1e9 - 35.128) < 0.01      # ViT-B/16 (cls)
    assert abs(O.flops_per_image(**bench.MODELS["vit_l16"]) / 1e9 - 123.109) < 0.05
    assert abs(O.flops_per_image(**bench.MODELS["vit_h14"]) / 1e9 - 310.867) < 0.1
    assert abs(O.flops_per_image(**bench.MODELS["vit_h14"], dim_head=80) / 1e9 - 334.590) < 0.1
    # NaViT config 5: 256 images / 83 901 tokens, block-diagonal attention 1.017 TFLOP
    sizes = bench.navit_sizes(256, 0)
    gemm, attn = bench.navit_flops(bench.MODELS["navit"], sizes)
    assert sum((h // 16) * (w // 16) for h, w in sizes) == 83901
    assert abs(attn / 1e12 - 1.017) < 0.002 and 12.8 < gemm / 1e12 < 13.3
