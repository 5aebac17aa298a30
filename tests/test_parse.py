from hpc_patterns_b200.utils.parse import main, parse_log, render

LOG = """+ export HPCP_DEVICE=0
# out_of_order | C C | Starting Benchmarking...
## out_of_order | C C | SUCCESS: Close from Theoretical Speedup
## out_of_order | C MD | FAILURE: Far from Theoretical Speedup
## in_order | C C | SUCCESS: Close from Theoretical Speedup
## in_order | C MD | FAILURE: Minimun Bandwish not reached
+ export HPCP_DEVICE=0 CUDA_DEVICE_MAX_CONNECTIONS=1
## fused | C  MD | SUCCESS: Close from Theoretical Speedup
"""


def test_parse_groups_by_env_commands_mode():
    t = parse_log(LOG)
    assert list(t) == ["HPCP_DEVICE=0", "HPCP_DEVICE=0 CUDA_DEVICE_MAX_CONNECTIONS=1"]
    assert t["HPCP_DEVICE=0"]["C C"] == {"out_of_order": "SUCCESS", "in_order": "SUCCESS"}
    assert t["HPCP_DEVICE=0"]["C MD"] == {"out_of_order": "FAILURE", "in_order": "FAILURE"}
    assert t["HPCP_DEVICE=0 CUDA_DEVICE_MAX_CONNECTIONS=1"]["C MD"] == {"fused": "SUCCESS"}


def test_render_has_one_table_per_env():
    text = render(parse_log(LOG))
    assert text.count("commands") == 2
    assert "out_of_order" in text and "in_order" in text and "fused" in text


def test_cli(tmp_path, capsys):
    p = tmp_path / "x.log"
    p.write_text(LOG)
    assert main([str(p), "github"]) == 0
    assert "| C C" in capsys.readouterr().out
    assert main([]) == 2


def test_roundtrip_with_real_driver_output(native):
    rc, out, _ = native.concurency_main(["nowait", "--commands", "C", "M2D", "--commands", "H2D", "D2H"],
                                        "fake:C=0.01,MD=0.0005,HD=0.0002,DH=0.0002,overlap=0.9")
    t = parse_log("export X=1\n" + out)
    assert t["X=1"]["C MD"]["nowait"] == "SUCCESS" and "HD DH" in t["X=1"]


def test_clock_summary_flags_throttle_reasons():
    from hpc_patterns_b200.utils.clocks import summarize

    lines = ["0, 1965, 1965, 950.0, Not Active, Not Active, Not Active, Active",
             "0, 1800, 1965, 980.0, Not Active, Not Active, Not Active, Active",
             "0, 210, 1965, 140.0, Not Active, Not Active, Not Active, Not Active",
             "garbage"]
    s = summarize(lines)
    assert s["sm_max_mhz"] == 1965 and s["reasons"] == ["sw_power_cap"] and s["samples"] == 3
    assert s["sm_mhz"] in (1800, 1882.5, 1965)   # median of the samples under load
    assert summarize([])["samples"] == 0


def test_report_tables(tmp_path):
    import json

    from hpc_patterns_b200.utils import report

    rows = [{"pattern": "peer2pear", "label": "x", "transport": "put", "engine": "tma", "ranks": 2, "bytes": 1024,
             "uni_GBps": 385.0, "bi_GBps": 700.0},
            {"pattern": "allreduce", "algo": "ring", "type": "float", "ranks": 8, "elements": 1 << 25, "ms": 1.2,
             "GBps_sent_per_rank": 770.0},
            {"pattern": "concurency", "backend": "fake", "mode": "fused", "commands": ["C", "DP"],
             "serial_total_us": 200, "concurrent_total_us": 105, "speedup": 1.9, "max_speedup": 2.0,
             "overlap_fraction": 0.95, "verdict": "SUCCESS"}]
    p = tmp_path / "rows.jsonl"
    p.write_text("\n".join(json.dumps(r) for r in rows) + "\nnot json\n")
    text = report.render(report.load_rows([str(p)]))
    assert "| 700.0 | 0.86 |" in text         # 385 / 450 per direction
    assert "| 770.0 | 1.71 |" in text         # 770 / 450
    assert "95%" in text and "SUCCESS" in text


def test_clock_sampler_without_a_driver_reports_no_samples():
    from hpc_patterns_b200.utils.clocks import ClockSampler

    import torch

    if torch.cuda.is_available():
        return  # covered by the GPU bench test
    s = ClockSampler(0).start().stop()
    assert s["samples"] == 0 and s["sm_mhz"] is None and s["reasons"] == []


def test_python_sweep_renders_tables_with_the_cpu_backend(native):
    """models.concurency.sweep == run_omp.sh in Python: env matrix x modes x groups -> tables."""
    from hpc_patterns_b200.models import concurency as cc

    text = cc.sweep(["nowait"], groups=[["C", "C"], ["C", "M2D"]], backend="cpu",
                    envs=[{}, {"OMP_NUM_THREADS": "2"}],
                    extra_args=["--repetitions", "2", "--tripcount_C", "2000", "--globalsize_C", "64",
                                "--globalsize_default_memory", "100000"])
    assert "OMP_NUM_THREADS=2" in text and "DEFAULT=1" in text
    assert text.count("nowait") >= 2 and ("SUCCESS" in text or "FAILURE" in text)
    total, per = cc.bench("serial", ["C", "M2D"], {"tripcount_C": 1000, "globalsize_C": 64,
                                                  "globalsize_M2D": 100000}, backend="cpu", n_repetitions=2)
    assert total > 0 and len(per) == 2
    total, per = cc.bench("nowait", ["C", "MD"], {"tripcount_C": 1000, "globalsize_C": 64,
                                                 "globalsize_MD": 100000}, backend="cpu", n_repetitions=2)
    assert total > 0 and per == []


def test_report_renders_tensor_parallel_and_gemm_rows(tmp_path):
    """Rows of `python -m hpc_patterns_b200 tp` and scripts/gemm_put_bench.py -> roofline tables."""
    import json

    from hpc_patterns_b200.utils import report

    rows = [{"ranks": 8, "m": 8192, "n": 8192, "k": 28672, "chunk": 2048,
             "row_parallel": {"fused_ms": 0.4, "stock_ms": 0.8, "speedup": 2.0},
             "row_parallel_allreduce": {"unavailable": "no multicast"},
             "column_parallel": {"fused_ms": 0.35, "stock_ms": 0.5, "speedup": 1.43}},
            {"m": 8192, "n": 8192, "k": 4096, "ranks": 2, "gemm_tflops": 1486.0,
             "cublas_tflops": 1662.0, "fused_gemm_put_ms": 0.401, "stock_cublas_then_memcpy_ms": 0.514}]
    p = tmp_path / "rows.jsonl"
    p.write_text("\n".join(json.dumps(r) for r in rows))
    text = report.render(report.load_rows([str(p)]))
    assert "## tensor-parallel layers" in text and "## tensor-core GEMM" in text
    line = [ln for ln in text.splitlines() if ln.startswith("| row_parallel (chunk 2048)")][0]
    cells = [c.strip() for c in line.split("|")]
    assert cells[2:6] == ["8", "8192", "8192", "28672"] and cells[8] == "2.00"
    assert "row_parallel_allreduce" not in text                      # unavailable rows are skipped
    assert "| 8192 | 8192 | 4096 | 2 | 1486 | 1662 | 1.50 |" in text     # 1486 / 989


def test_clock_sampler_nvml_thread_with_a_fake_driver(monkeypatch):
    """The NVML polling thread against a fake pynvml: handle by UUID, samples only while resumed (the bench keeps it
    paused outside timed regions), throttle-reason bits decoded, median over the samples taken under load."""
    import sys
    import time
    import types

    from hpc_patterns_b200.utils.clocks import ClockSampler

    state = {"clock": 1965, "power_mw": 900_000, "mask": 0, "by_uuid": 0, "by_index": 0, "reads": 0}
    nv = types.ModuleType("pynvml")
    nv.NVML_CLOCK_SM = 1
    nv.nvmlInit = lambda: None

    def by_uuid(u):
        state["by_uuid"] += 1
        assert u == b"GPU-1234"
        return "handle"

    def by_index(i):
        state["by_index"] += 1
        return "handle"

    def clock(h, kind):
        state["reads"] += 1
        return state["clock"]
    nv.nvmlDeviceGetHandleByUUID, nv.nvmlDeviceGetHandleByIndex = by_uuid, by_index
    nv.nvmlDeviceGetMaxClockInfo = lambda h, kind: 1965
    nv.nvmlDeviceGetClockInfo = clock
    nv.nvmlDeviceGetPowerUsage = lambda h: state["power_mw"]
    nv.nvmlDeviceGetCurrentClocksEventReasons = lambda h: state["mask"]
    monkeypatch.setitem(sys.modules, "pynvml", nv)

    s = ClockSampler(gpu_index=3, period_ms=0.2, uuid="GPU-1234").start(paused=True)
    assert state["by_uuid"] == 1 and state["by_index"] == 0
    time.sleep(0.05)
    assert state["reads"] == 0, "paused: no NVML call may happen next to a timed region's barrier"
    s.resume()
    time.sleep(0.05)
    state.update(clock=1800, mask=0x4)          # sw_power_cap appears while under load
    time.sleep(0.05)
    s.pause()
    time.sleep(0.01)
    n = state["reads"]
    state.update(clock=210, power_mw=140_000, mask=0x8)   # idle again, and a reason that must NOT be recorded now
    time.sleep(0.05)
    assert state["reads"] == n
    out = s.stop()
    assert out["sampler"] == "nvml-thread" and out["samples"] == n > 10
    assert out["sm_max_mhz"] == 1965 and out["sm_mhz"] in (1800, 1882.5, 1965)
    assert out["reasons"] == ["sw_power_cap"] and out["power_w_max"] == 900.0
