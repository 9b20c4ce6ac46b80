"""The odometry and training measurement scripts under scripts/ on a machine without a GPU: their flags, their refusal
to run without a device, that they share code only through scripts/measure.py, and measure's pure functions."""
import ast
import json
import os
import re
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SCRIPTS = os.path.join(ROOT, "scripts")

# every script's flags; the output flag is --json FILE or --out DIR
FLAGS = {
    "gpu_odometry_capi": {"--frames", "--json"},
    "gpu_odometry_train_capi": {"--batch", "--h", "--out", "--rounds", "--w", "--warmup"},
    "gpu_odometry_normalized": {"--json", "--samples"},
    "gpu_odometry_streams": {"--out", "--profile", "--profile_sizes", "--seconds"},
    "gpu_odometry_eval": {"--out", "--samples", "--seconds"},
    "gpu_odometry_streams_normalized": {"--out", "--samples", "--seconds"},
    "gpu_odometry_streams_pre": {"--out", "--samples", "--seconds"},
    "gpu_odometry_streams_info": {"--out", "--samples", "--seconds"},
    "gpu_odometry_streams_pre_adapt_info": {"--out", "--samples", "--seconds"},
    "gpu_odometry_streams_adapt": {"--out", "--samples", "--seconds"},
    "gpu_odometry_streams_adapt_geometries": {"--out", "--samples", "--seconds"},
    "gpu_odometry_streams_adapt_geometries_info": {"--out", "--samples", "--seconds"},
    "gpu_odometry_streams_adapt_group": {"--gpus", "--out", "--samples", "--seconds"},
    "gpu_train_dropout": {"--out", "--replays", "--rounds", "--warmup"},
    "gpu_train_geometries": {"--configs", "--out", "--samples", "--seconds"},
    "gpu_train_group": {"--batch", "--gpus", "--out", "--samples", "--seconds"},
    "gpu_train_pre_normals": {"--batches", "--out", "--replays", "--reps", "--rounds", "--warmup"},
}
NO_GPU = ("needs a GPU", "no CUDA device")


def _run(args):
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    return subprocess.run([sys.executable] + args, cwd=ROOT, env=env, capture_output=True, text=True, timeout=600)


@pytest.fixture(scope="module")
def runs(tmp_path_factory):
    """{script: (`--help` run, run without a GPU, its output path)}, the runs made side by side."""
    out = tmp_path_factory.mktemp("out")
    jobs = {}
    for s, flags in FLAGS.items():
        path = str(out / s / ("result.json" if "--json" in flags else "dir"))
        flag = "--json" if "--json" in flags else "--out"
        jobs[s] = ([os.path.join(SCRIPTS, s + ".py"), "--help"], [os.path.join(SCRIPTS, s + ".py"), flag, path], path)
    with ThreadPoolExecutor(max_workers=min(8, os.cpu_count() or 1)) as pool:
        done = {s: (pool.submit(_run, h), pool.submit(_run, r), p) for s, (h, r, p) in jobs.items()}
        return {s: (h.result(), r.result(), p) for s, (h, r, p) in done.items()}


@pytest.mark.parametrize("script", sorted(FLAGS))
def test_help_lists_the_flags(runs, script):
    r = runs[script][0]
    assert r.returncode == 0, r.stderr
    usage = r.stdout.split("\n\n")[0]
    assert set(re.findall(r"--\w+", usage)) == FLAGS[script]


@pytest.mark.parametrize("script", sorted(FLAGS))
def test_no_gpu_fails_and_writes_nothing(runs, script):
    _, r, path = runs[script]
    assert r.returncode != 0
    assert any(m in r.stderr for m in NO_GPU), r.stderr
    assert not os.path.exists(path)


@pytest.mark.parametrize("script", sorted(FLAGS))
def test_imports_no_other_script(script):
    tree = ast.parse(open(os.path.join(SCRIPTS, script + ".py")).read())
    modules = set()
    for node in ast.walk(tree):
        if isinstance(node, ast.Import):
            modules |= {a.name.split(".")[0] for a in node.names}
        elif isinstance(node, ast.ImportFrom) and node.module:
            modules.add(node.module.split(".")[0])
    assert not modules & set(FLAGS), modules & set(FLAGS)


@pytest.fixture(scope="module")
def measure():
    sys.path.insert(0, SCRIPTS)
    try:
        import measure
    finally:
        sys.path.remove(SCRIPTS)
    return measure


def test_summary(measure):
    assert measure.summary([3.0, 1.0, 2.0, 5.0]) == {"median": 2.5, "min": 1.0, "max": 5.0}
    assert measure.summary([4.0]) == {"median": 4.0, "min": 4.0, "max": 4.0}


def test_paired(measure):
    d, med = measure.paired([1.0, 2.0, 4.0], [1.5, 2.0, 7.0])
    assert d == [0.5, 0.0, 3.0] and med == 0.5
    d, med = measure.paired([1.0, 1.0], [2.0, 4.0])
    assert d == [1.0, 3.0] and med == 2.0


def test_emit_prints_what_it_writes(measure, tmp_path, capsys):
    res = {"gpu_before": "unavailable", "sizes": {"64x720": {"n_stride": 7, "ms": [0.25, 0.5]}}, "ok": True}
    path = tmp_path / "new" / "result.json"
    measure.emit(res, str(path))
    printed = capsys.readouterr().out
    assert printed == path.read_text() + "\n"
    assert printed == json.dumps(res, indent=1) + "\n"
    measure.emit(res, "")
    assert capsys.readouterr().out == printed
