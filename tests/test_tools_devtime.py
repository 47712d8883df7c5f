"""tools/devtime.py, the one device timer, host timer and card reading every measurement tool uses, and the rule that
keeps it the only one: no other tool builds a CUDA event pair (except where a comment says why it cannot use
device_ms) or runs nvidia-smi."""
import glob
import math
import os
import py_compile
import re
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOOLS = os.path.join(ROOT, "tools")
sys.path.insert(0, TOOLS)
import devtime  # noqa: E402

SCRIPTS = sorted(glob.glob(os.path.join(TOOLS, "*.py")))


@pytest.mark.parametrize("path", SCRIPTS, ids=os.path.basename)
def test_tool_compiles(path, tmp_path):
    py_compile.compile(path, cfile=str(tmp_path / "x.pyc"), doraise=True)


def test_only_devtime_times_and_reads_the_card():
    for path in SCRIPTS:
        if os.path.basename(path) == "devtime.py":
            continue
        with open(path) as fh:
            lines = fh.read().splitlines()
        name = os.path.basename(path)
        assert not any("nvidia-smi" in ln for ln in lines), f"{name} reads the card itself; use devtime.card()"
        for i, ln in enumerate(lines):
            if "Event(enable_timing" in ln:
                above = [a for a in lines[max(0, i - 3):i] if a.strip().startswith("#")]
                assert any("device_ms" in a for a in above), \
                    f"{name}:{i + 1} builds its own event pair without a comment saying why device_ms does not fit"


def _fake_smi(tmp_path, monkeypatch, body):
    exe = tmp_path / "nvidia-smi"
    exe.write_text("#!/bin/sh\n" + body)
    exe.chmod(0o755)
    monkeypatch.setenv("PATH", f"{tmp_path}{os.pathsep}{os.environ.get('PATH', '')}")


def test_card_gives_error_text_when_nvidia_smi_fails(tmp_path, monkeypatch):
    _fake_smi(tmp_path, monkeypatch, "echo 'no devices were found' >&2\nexit 6\n")
    c = devtime.card()
    assert set(c) == {"name", "power_limit_w", "sm_clock_max_mhz"}
    assert len(set(c.values())) == 1
    err = c["name"]
    assert isinstance(err, str) and "nvidia-smi" in err and "6" in err
    assert devtime.card_line(c) == err


def test_card_reads_one_device_and_only_queries(tmp_path, monkeypatch):
    args = tmp_path / "args"
    _fake_smi(tmp_path, monkeypatch, f'printf "%s\\n" "$@" > {args}\necho "NVIDIA H100 80GB HBM3, 700.00, 1980"\n')
    c = devtime.card()
    assert c == {"name": "NVIDIA H100 80GB HBM3", "power_limit_w": 700.0, "sm_clock_max_mhz": 1980.0}
    assert devtime.card_line(c) == "NVIDIA H100 80GB HBM3, power limit 700 W, max SM clock 1980 MHz"
    for a in args.read_text().split():
        assert re.fullmatch(r"--(id=GPU-[0-9a-f-]+|query-gpu=name,power\.limit,clocks\.max\.sm|format=csv,noheader,nounits)",
                            a), a


@pytest.mark.parametrize("warmup,reps", [(0, 1), (1, 7), (3, 20)])
def test_host_ms_calls_fn_warmup_plus_reps_times(warmup, reps):
    calls = []
    ms = devtime.host_ms(lambda: calls.append(1), reps=reps, warmup=warmup)
    assert len(calls) == warmup + reps
    assert ms >= 0.0 and math.isfinite(ms)


def test_host_ms_min_s_runs_until_the_clock_passes_it():
    calls = []
    ms = devtime.host_ms(lambda: calls.append(1), warmup=1, min_s=0.02)
    assert len(calls) >= 2
    assert ms * (len(calls) - 1) >= 0.02 * 1e3


def test_host_ms_takes_reps_or_min_s():
    with pytest.raises(ValueError):
        devtime.host_ms(lambda: None)
    with pytest.raises(ValueError):
        devtime.host_ms(lambda: None, reps=3, min_s=0.1)


def test_device_ms_raises_without_a_device(monkeypatch):
    monkeypatch.setattr(devtime.torch.cuda, "is_available", lambda: False)
    calls = []
    with pytest.raises(RuntimeError, match="CUDA device"):
        devtime.device_ms(lambda: calls.append(1), 5, 2)
    assert calls == []


@pytest.mark.gpu
def test_device_ms_times_fn_on_the_device():
    import torch
    x = torch.ones(1 << 20, device="cuda")
    calls = []

    def fn():
        calls.append(1)
        x.mul_(1.0)
    ms = devtime.device_ms(fn, 20, 3)
    assert len(calls) == 23
    assert ms > 0.0 and math.isfinite(ms)
