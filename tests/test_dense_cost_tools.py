"""The whole-run voxel map cost tools: every tools/dense_* script imports, and the shared module's summary statistics
and card report behave as the scripts' JSON needs them to."""
import glob
import importlib
import os
import subprocess
import sys

import pytest

TOOLS = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools")
if TOOLS not in sys.path:
    sys.path.insert(0, TOOLS)

import dense_cost  # noqa: E402

SCRIPTS = sorted(os.path.basename(p)[:-3] for p in glob.glob(os.path.join(TOOLS, "dense_*.py"))
                 if os.path.basename(p) != "dense_cost.py")


@pytest.mark.parametrize("name", SCRIPTS)
def test_script_imports(name, monkeypatch):
    monkeypatch.setattr(sys, "dont_write_bytecode", sys.dont_write_bytecode)  # the scripts set it on import
    assert callable(importlib.import_module(name).main)


def test_stats():
    assert dense_cost.stats([0.5, 3.14159, 2.0, 10.123456]) == {"median": 2.5708, "min": 0.5, "max": 10.1235}


def test_gpu_info_from_nvidia_smi(monkeypatch):
    monkeypatch.setitem(sys.modules, "pynvml", None)

    def run(cmd, **kw):
        assert cmd == ["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"]
        return subprocess.CompletedProcess(cmd, 0, stdout="NVIDIA H100 80GB HBM3, 700.00\nNVIDIA H100 80GB HBM3, 500.00\n")

    monkeypatch.setattr(dense_cost.subprocess, "run", run)
    assert dense_cost.gpu_info() == {"name": "NVIDIA H100 80GB HBM3", "power_limit_w": 700.0}


def test_gpu_info_without_nvml_or_nvidia_smi(monkeypatch, tmp_path):
    import torch
    monkeypatch.setitem(sys.modules, "pynvml", None)
    monkeypatch.setenv("PATH", str(tmp_path))
    monkeypatch.setattr(torch.cuda, "get_device_name", lambda index=None: "some card")
    assert dense_cost.gpu_info() == {"name": "some card", "power_limit_w": None}
