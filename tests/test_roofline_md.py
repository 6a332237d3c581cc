"""``tools/roofline_md.py`` renders the committed site-profile / all-reduce JSON into the tables of a ROOFLINE.md."""
import json
import os

from tools import roofline_md

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_roofline_md_renders_sites_and_collectives(tmp_path):
    site = {"peak_bf16_flops": 1.6946e15, "peak_hbm_Bps": 6.5719e12, "ours_ms": 10.0, "roofline_ms": 6.0,
            "sites": [{"site": "gemm M128 N256 K64", "calls": 3, "us": 1500.0, "tflops": 900.0, "gbps": 1200.0, "bound": "compute",
                       "frac_of_roofline": 0.53},
                      {"site": "swiglu_fwd", "calls": 2, "us": 500.0, "tflops": 0.0, "gbps": 4700.0, "bound": "memory", "frac_of_roofline": None}],
            "other": [["void at::native::reduce_kernel<512>", 91.0, 1], ["Memset", 16.0, 11]]}
    ar = [{"kbytes": 65536, "n_gpus": 8, "nccl_us": 275.0, "p2p_us": 204.0, "nvls_us": 201.0, "nccl_busGBs": 427.0, "p2p_busGBs": 576.0,
           "nvls_busGBs": 584.0},
          {"fused_update": "llama_250m", "n_gpus": 8, "params": 98888192, "transport": "nvls", "us": 697.0, "link_GBs_per_direction": 496.0,
           "roofline_us_at_770GBs": 449.0, "fraction_of_roofline": 0.64}]
    sp, ap, out = tmp_path / "site.json", tmp_path / "ar.json", tmp_path / "ROOFLINE.md"
    sp.write_text(json.dumps(site)); ap.write_text(json.dumps(ar))
    roofline_md.main(["--site", f"toy model={sp}", "--allreduce", str(ap), str(tmp_path / "missing.json"), "--out", str(out)])
    text = out.read_text()
    assert "### toy model" in text and "1694.6 TFLOP/s burst, 6571.9 GB/s" in text
    assert "| `gemm M128 N256 K64` | 3 | 1.500 | 900 | 1200 | compute | 0.53 |" in text
    assert "| `swiglu_fwd` | 2 | 0.500 | 0 | 4700 | memory | 0.00 |" in text          # a missing fraction renders as 0.00
    assert "reduce_kernel<512>` 0.09 ms" in text and "Memset" not in text           # only library kernels above 0.05 ms are listed
    assert "| 8 | 65536 | 427 (275 µs) | 576 (204 µs) | 584 (201 µs) | 0.76 |" in text
    assert "| llama_250m (98.9 M) | 8 | nvls | 697 | 496 | 449 | 0.64 |" in text
