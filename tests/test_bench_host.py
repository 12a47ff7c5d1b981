"""Host-side logic of bench.py and of the lazy batch outputs (no GPU)."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import ROOT

sys.path.insert(0, ROOT)
import bench  # noqa: E402


def test_algorithmic_bytes_match_baseline_md():
    # BASELINE.md §3: N=10 000, D=512, C=2 -> 20.99 MB; 2048 + 8C bytes per patch + 341 008 B of weights
    b = bench.algorithmic_bytes_fwd(10000, 512, 2)
    assert b == 10000 * (2048 + 16) + 341008 + 4 * 2 * 512 + 4 * 2
    assert abs(b / 1e6 - 20.99) < 0.01


def test_warmup_is_rank_invariant_under_torchrun():
    """Every bench step contains two all-gathers when WORLD_SIZE > 1: a time-based warm-up count differs
    between ranks and deadlocks them."""
    for world in (2, 4, 8):
        fixed, timed, extra = bench.warmup_plan(world, 3)
        assert timed == 0.0 and fixed >= 3 and extra > 0
    fixed, timed, extra = bench.warmup_plan(1, 0)
    assert fixed >= 3 and timed > 0 and extra == 0          # W >= 3 even if the caller asks for less


def test_clock_sampler_parses_nvidia_smi_rows():
    s = bench.ClockSampler()
    s.proc = object.__new__(subprocess.Popen)               # pretend a sampler ran
    s.proc.terminate = lambda: None
    s.proc.wait = lambda timeout=None: 0
    s.rows = ["1965, 1965, 612.3, Not Active, Not Active, Not Active, Active",
              "1800, 1965, 998.0, Not Active, Not Active, Not Active, Not Active", "garbage"]
    out = s.stop()
    assert out["sm_mhz"] == 1882.5 and out["sm_max_mhz"] == 1965.0 and out["reasons"] == ["sw_power_cap"]
    assert out["samples"] == 2


def test_reference_arm_prints_the_contract_line():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--steps", "1",
                        "--warmup", "1", "--ref-bags", "1"], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-500:]
    d = json.loads(r.stdout.strip().splitlines()[-1])
    for k in ("impl", "metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better",
              "scaling", "vs_baseline", "dtype", "data", "config", "cpu_baseline", "e2e", "gpu_launches"):
        assert k in d, k
    from oracle import stage_ref
    kind = "reference" if stage_ref.staged("dsmil.py") else "port"      # the unmodified module when build() staged it
    assert d["impl"] == "reference" and d["vs_baseline"] is None and d["cpu_baseline"]["kind"] == kind
    assert d["e2e"]["h2d_bytes_per_step"] == 0 and d["e2e"]["value"] == d["value"] and d["value"] > 0


def test_reference_arm_other_ranks_exit_quietly():
    env = dict(os.environ, RANK="1", WORLD_SIZE="2", LOCAL_RANK="1")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--gpus", "2",
                        "--steps", "1", "--warmup", "1"], capture_output=True, text=True, timeout=300, env=env)
    assert r.returncode == 0 and r.stdout.strip() == ""


def test_bag_outputs_lazy_sequence():
    from dsmil_wsi_b200.functional import BagOutputs
    Ns = [3, 1, 5]
    classes = torch.arange(18.).view(9, 2); A = classes + 100
    pred = torch.arange(6.).view(3, 2); B = torch.arange(24.).view(3, 2, 4)
    o = BagOutputs(classes, pred, A, B, Ns)
    assert len(o) == 3 and o.packed[0] is classes
    c, p, a, b = o[1]
    assert torch.equal(c, classes[3:4]) and torch.equal(p, pred[1:2]) and torch.equal(a, A[3:4]) and torch.equal(b, B[1:2])
    assert torch.equal(o[-1][0], classes[4:9]) and len(o[0:2]) == 2 and len(list(o)) == 3
    with pytest.raises(IndexError):
        o[3]
    assert c.data_ptr() == classes[3:4].data_ptr()          # views, not copies
