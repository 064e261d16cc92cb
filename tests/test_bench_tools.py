"""The engine-option benchmarks under tools/ without a GPU: every script built on tools/benchlib.py parses its arguments, and
benchlib's alternation and record writer keep their order and format."""
import importlib.util
import json
import os
import re
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOOLS = os.path.join(ROOT, "tools")
SCRIPTS = sorted(f for f in os.listdir(TOOLS) if f.endswith(".py") and f != "benchlib.py"
                 and re.search(r"^(from benchlib import|import benchlib)", open(os.path.join(TOOLS, f)).read(), re.M))


def _benchlib():
    spec = importlib.util.spec_from_file_location("benchlib", os.path.join(TOOLS, "benchlib.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_the_option_benchmarks_use_benchlib():
    assert "class_bench.py" in SCRIPTS and len(SCRIPTS) >= 12, SCRIPTS


@pytest.mark.parametrize("script", SCRIPTS)
def test_script_help(script):
    p = subprocess.run([sys.executable, os.path.join(TOOLS, script), "--help"], cwd=ROOT, capture_output=True, text=True, timeout=120)
    assert p.returncode == 0, p.stderr
    assert "usage:" in p.stdout


def test_alternate_runs_off_then_on():
    calls = []
    _benchlib().alternate(3, lambda run, on: calls.append((run, on)))
    assert calls == [(0, False), (0, True), (1, False), (1, True), (2, False), (2, True)]
    calls.clear()
    _benchlib().alternate(0, lambda run, on: calls.append((run, on)))
    assert calls == []


def test_card_queries_name_power_limit_and_clocks(monkeypatch):
    bl = _benchlib()
    seen = []
    monkeypatch.setattr(bl.subprocess, "run", lambda cmd, **kw: seen.append(cmd) or subprocess.CompletedProcess(cmd, 0, " H100, 700 W \n", ""))
    assert bl.card() == "H100, 700 W"
    assert seen == [["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"]]


def test_recorder_writes_card_lines_around_the_records(monkeypatch, tmp_path, capsys):
    bl = _benchlib()
    cards = iter(["card before", "card after"])
    monkeypatch.setattr(bl, "card", lambda: next(cards))
    out = bl.Recorder("x_bench", str(tmp_path / "out"), workload="W")
    out.record({"run": 0, "on": False, "ms": [1.5, 2]})
    out.record({"run": 0, "on": True, "nested": {"a": None}})
    out.finish()
    want = [{"gpu": "card before", "fields": bl.CARD_FIELDS, "workload": "W"}, {"run": 0, "on": False, "ms": [1.5, 2]},
            {"run": 0, "on": True, "nested": {"a": None}}, {"gpu_after": "card after"}]
    assert os.listdir(tmp_path / "out") == ["x_bench.jsonl"]
    lines = (tmp_path / "out" / "x_bench.jsonl").read_text().splitlines()
    assert [json.loads(x) for x in lines] == want
    assert [list(json.loads(x)) for x in lines] == [list(x) for x in want]
    assert capsys.readouterr().out.splitlines() == lines


def test_recorder_without_out_dir_only_prints(monkeypatch, tmp_path, capsys):
    bl = _benchlib()
    monkeypatch.setattr(bl, "card", lambda: "card")
    monkeypatch.chdir(tmp_path)
    out = bl.Recorder("x_bench")
    out.record({"k": 1})
    out.finish()
    assert os.listdir(tmp_path) == []
    assert [json.loads(x) for x in capsys.readouterr().out.splitlines()] == [{"gpu": "card", "fields": bl.CARD_FIELDS}, {"k": 1},
                                                                             {"gpu_after": "card"}]
