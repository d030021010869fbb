"""Host-side helpers of bench.py / tools (no GPU needed)."""
import importlib.util
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _load(path, name):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_clock_sampler_parsing():
    bench = _load(os.path.join(ROOT, "bench.py"), "bench_mod")
    s = bench.ClockSampler(2)
    s.proc = type("P", (), {"terminate": lambda self: None, "wait": lambda self, timeout=None: 0, "kill": lambda self: None})()
    s.t_mark = 100.0
    s.lines = [(101.0 + i, ln) for i, ln in enumerate([
        "0, 1965, 1965, 512.3, Not Active, Not Active, Not Active, Active",
        "1, 1800, 1965, 700.0, Not Active, Not Active, Not Active, Not Active",
        "2, 300, 1965, 90.0, Active, Not Active, Not Active, Not Active",      # GPU outside the job: ignored
        "garbage line",
        "0, 1900, 1965, 650.0, Not Active, Not Active, Not Active, Active",
    ])]
    s.lines.insert(0, (50.0, "0, 400, 1965, 90.0, Not Active, Not Active, Not Active, Not Active"))   # before the timed region: ignored
    out = s.stop()
    assert out["sm_mhz"] == 1900 and out["sm_max_mhz"] == 1965 and out["samples"] == 3
    assert out["reasons"] == ["sw_power_cap"] and out["power_w_max"] == 700.0 and out["scope"] == "timed region"
    # a timed region too short to be sampled (8 GPUs, ~0.2 s): the loaded warm-up samples are reported instead of `null`
    s2 = bench.ClockSampler(2)
    s2.proc = s.proc
    s2.t_mark = 200.0
    s2.lines = [(150.0, "0, 1700, 1965, 800.0, Not Active, Not Active, Not Active, Active"),
                (150.1, "1, 1710, 1965, 810.0, Not Active, Not Active, Not Active, Active")]
    out2 = s2.stop()
    assert out2 is not None and out2["samples"] == 2 and out2["scope"] == "warm-up + timed region"


def test_model_kwargs_and_metric_config():
    bench = _load(os.path.join(ROOT, "bench.py"), "bench_mod2")
    kw = bench.model_kwargs("llama125m")
    assert kw["vocab_size"] == 50257 and kw["hidden_size"] == 768 and kw["num_key_value_heads"] == 12
    assert "tokens/sec" in bench.METRIC


def test_reference_arm_reports_unavailable_instead_of_crashing(monkeypatch, capsys):
    """Without a GPU (or without the install) `--impl reference` must print a JSON line and exit 0."""
    bench = _load(os.path.join(ROOT, "bench.py"), "bench_mod3")
    args = type("A", (), dict(steps=2, warmup=1, model="llama125m", batch=2, seq=16, n_acc=1))()
    out = bench.run_reference_arm(args)
    assert out["impl"] == "reference"
    assert "unavailable" in out or "value" in out


def test_launch_summary_parses_ncu_csv(tmp_path, capsys):
    ls = _load(os.path.join(ROOT, "tools", "launch_summary.py"), "launch_summary")
    csv = ('==PROF== noise\n"ID","Process ID","Process Name","Host Name","Kernel Name","Context","Stream","Block Size","Grid Size","Device","CC",'
           '"Section Name","Metric Name","Metric Unit","Metric Value"\n'
           '"0","1","python","h","void acco::ce_fwd_kernel(const __nv_bfloat16 *)","1","7","(512, 1, 1)","(8192, 1, 1)","0","10.0","Command line profiler metrics","gpu__time_duration.sum","us","140.5"\n'
           '"1","1","python","h","void acco::ce_fwd_kernel(const __nv_bfloat16 *)","1","7","(512, 1, 1)","(8192, 1, 1)","0","10.0","Command line profiler metrics","gpu__time_duration.sum","us","139.5"\n'
           '"2","1","python","h","nvjet_tst_192x256","1","7","(384, 1, 1)","(148, 1, 1)","0","10.0","Command line profiler metrics","gpu__time_duration.sum","ns","20000"\n')
    p = tmp_path / "l.csv"
    p.write_text(csv)
    sys.argv = ["launch_summary.py", str(p)]
    ls.main()
    out = capsys.readouterr().out
    assert "3 launches, total 0.300 ms" in out and "x2" in out and "ce_fwd_kernel" in out


def test_memory_plan_tool():
    """tools/memory_plan.py: persistent buffers follow the arena / optimizer layout (2 x 2 bytes of bf16 parameters and 2 x 2 bytes of
    bf16 gradient accumulators per parameter, 16 bytes / W of fp32 shard).  The shipped 8-GPU fine-tuning job (Llama-3.2-1B) fits an
    80 GB H100; Llama-3-8B does not fit on 8 of them even before activations (80.3 GB of persistent buffers per GPU)."""
    import importlib.util
    import os
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    spec = importlib.util.spec_from_file_location("memory_plan", os.path.join(root, "tools", "memory_plan.py"))
    mp = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mp)
    p8 = mp.main(["--model", "llama3-1b", "--gpus", "8", "--batch", "4", "--seq", "512"])
    assert p8["fits_80gb"] and 5 < p8["total_gb"] < 40
    assert abs(p8["buffers_gb"]["optimizer shard: master, exp_avg, exp_avg_sq, stash (fp32)"] - 16 * p8["size_slice"] / 1e9) < 1e-9
    big = mp.main(["--model", "llama3-8b", "--gpus", "8", "--batch", "4", "--seq", "512"])
    assert big["parameters"] == 8_030_261_248 and not big["fits_80gb"]
    persistent = sum(v for k, v in big["buffers_gb"].items() if not k.startswith("activations"))
    assert persistent > 0.92 * 80
