"""CPU checks of tests/option_guard.py: the option table it reads from host.h is the one the library has, the defaults it
reads are what a fresh process starts with, options() restores on every exit, and every GPU test module uses the guard."""
import ast
import glob
import json
import os
import subprocess
import sys

import pytest

import pigo_b200
from option_guard import DEFAULTS, HOST_H, options, options_at_defaults, parse_options, snapshot   # noqa: F401

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_parsed_names_are_the_options_the_library_accepts():
    assert len(DEFAULTS) >= 40
    for name, default in DEFAULTS.items():
        with options(**{name: default + 3}):
            assert pigo_b200.get_option(name) == default + 3, name
        assert pigo_b200.get_option(name) == default, name
    with pytest.raises(pigo_b200.PigoError):
        pigo_b200.set_option("no_such_option", 1)
    with pytest.raises(KeyError):
        with options(no_such_option=1):
            pass


def test_a_fresh_process_starts_with_the_parsed_defaults():
    code = ("import json, sys, pigo_b200; names = json.loads(sys.argv[1]); "
            "print(json.dumps({n: pigo_b200.get_option(n) for n in names}))")
    r = subprocess.run([sys.executable, "-c", code, json.dumps(sorted(DEFAULTS))], cwd=ROOT, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    assert json.loads(r.stdout.strip().splitlines()[-1]) == DEFAULTS


def test_options_restores_every_option_on_exception():
    before = snapshot()
    with pytest.raises(RuntimeError):
        with options(tile_ks=7, queue_cap=16):
            pigo_b200.set_option("gather_limit", 4)     # set in the body, not through options(): restored as well
            assert pigo_b200.get_option("tile_ks") == 7
            raise RuntimeError("inside")
    assert snapshot() == before


@pytest.fixture
def option_set_by_a_fixture():
    with options(tile_ks=9):
        yield


def test_the_guard_checks_after_the_tests_own_fixtures(option_set_by_a_fixture):
    """The guard is an autouse fixture of the module, so pytest sets it up before the fixtures a test asks for and tears it
    down after them: an option a fixture restores at its teardown is not reported."""
    assert pigo_b200.get_option("tile_ks") == 9


def test_parser_rejects_a_member_without_default_or_outside_the_table():
    text = open(HOST_H).read()
    anchor = "  std::atomic<long long> timing{0};"
    assert anchor in text
    with pytest.raises(ValueError, match="without an integer default"):
        parse_options(text.replace(anchor, anchor + "\n  std::atomic<long long> new_knob;"))
    with pytest.raises(ValueError, match="new_knob"):
        parse_options(text.replace(anchor, anchor + "\n  std::atomic<long long> new_knob{3};"))
    assert parse_options(text) == DEFAULTS


def _marked_gpu(tree: ast.Module) -> bool:
    """Module-level `pytestmark = ...` or any decorator / mark that names pytest.mark.gpu."""
    for node in ast.walk(tree):
        if isinstance(node, ast.Attribute) and node.attr == "gpu" and isinstance(node.value, ast.Attribute) and node.value.attr == "mark":
            return True
    return False


def _imports_guard(tree: ast.Module) -> bool:
    return any(isinstance(n, ast.ImportFrom) and n.module == "option_guard" and any(a.name == "options_at_defaults" and a.asname is None
                                                                                    for a in n.names)
               for n in tree.body)


def test_every_gpu_module_imports_the_guard():
    gpu_modules, missing = [], []
    for path in sorted(glob.glob(os.path.join(ROOT, "tests", "test_*.py"))):
        tree = ast.parse(open(path).read(), filename=path)
        if _marked_gpu(tree):
            gpu_modules.append(os.path.basename(path))
            if not _imports_guard(tree):
                missing.append(os.path.basename(path))
    assert "test_gpu_parity.py" in gpu_modules and len(gpu_modules) >= 9
    assert missing == [], f"GPU test modules without `from option_guard import options_at_defaults`: {missing}"
