"""CPU: the scripts under tools/ compile, import only names the package has, and measure through tools/_harness.py: no script
but the harness queries nvidia-smi or makes timing events, and every script on the harness prints the card it measured on."""
import ast
import glob
import importlib
import os
import re
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
SCRIPTS = sorted(glob.glob(os.path.join(ROOT, "tools", "*.py")))
# train_dp.py runs one process per GPU under torch.distributed.run and times each rank's own device
OWN_CLOCK = {"_harness.py", "train_dp.py"}


def _source(path):
    with open(path) as fh:
        return fh.read()


ON_HARNESS = [p for p in SCRIPTS if "from _harness import" in _source(p)]


def _called(nodes, name):
    return any(isinstance(n, ast.Call) and getattr(n.func, "id", getattr(n.func, "attr", None)) == name
               for node in nodes for n in ast.walk(node))


@pytest.mark.parametrize("path", SCRIPTS, ids=os.path.basename)
def test_script_compiles(path):
    compile(_source(path), path, "exec")


@pytest.mark.parametrize("path", SCRIPTS, ids=os.path.basename)
def test_script_imports_resolve(path):
    """Every `from dmnerf_b200... import X` and `from _harness import X` names something that exists: a script whose imports
    went stale after an API change fails here, not on the GPU."""
    for node in ast.walk(ast.parse(_source(path))):
        if not (isinstance(node, ast.ImportFrom) and node.module and node.module.split(".")[0] in ("dmnerf_b200", "_harness")):
            continue
        module = importlib.import_module(node.module)
        for alias in node.names:
            if not hasattr(module, alias.name):             # else a submodule, or the import fails
                importlib.import_module(node.module + "." + alias.name)


@pytest.mark.parametrize("path", [p for p in SCRIPTS if os.path.basename(p) not in OWN_CLOCK], ids=os.path.basename)
def test_script_measures_through_the_harness(path):
    src = _source(path)
    assert "nvidia-smi" not in src, "query the card with _harness.gpu_identity"
    assert "enable_timing" not in src, "time with _harness.event_ms or _harness.alternate"


def test_harness_runs_only_the_read_only_card_query():
    src = _source(os.path.join(ROOT, "tools", "_harness.py"))
    assert re.findall(r"--[\w-]+", src) == ["--query-gpu", "--format"]
    assert re.findall(r"--query-gpu=[\w.,]+", src) == ["--query-gpu=name,power.limit"]


@pytest.mark.parametrize("path", ON_HARNESS, ids=os.path.basename)
def test_script_on_the_harness_prints_the_card(path):
    """The scope (a function, or the module's own statements) that prints the result also reads gpu_identity."""
    tree = ast.parse(_source(path))
    scopes = [[n] for n in ast.walk(tree) if isinstance(n, ast.FunctionDef)]
    scopes.append([n for n in tree.body if not isinstance(n, (ast.FunctionDef, ast.ClassDef))])
    printing = [s for s in scopes if _called(s, "print")]
    assert printing, "no print"
    assert all(_called(s, "gpu_identity") for s in printing), "a scope prints without gpu_identity"
