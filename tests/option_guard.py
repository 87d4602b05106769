"""The library's tuning options (`struct Options`, pigo_b200/csrc/host.h) are process-global, so an option a test sets and
does not restore changes which kernels every later test runs, while the oracle comparison keeps passing.  This module
reads the option table and its defaults from host.h (no hand-written copy) and gives the tests:

  options(**overrides)   context manager: snapshots every option, applies the overrides, restores every option
  options_at_defaults    autouse fixture: after each test (after the test's own fixtures), every option must be back
                         at its default; if not, all are reset and the test that leaked fails, naming the options

Every module marked `gpu` imports `options_at_defaults` (tests/test_option_guard.py checks that)."""
import contextlib
import os
import re

import pytest

import pigo_b200

HOST_H = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "pigo_b200", "csrc", "host.h")


def parse_options(text: str) -> dict:
    """{option name: default} from the text of host.h: the names of the find() table, the defaults of the member
    initialisers.  Raises ValueError if a member has no integer initialiser or the table and the members differ."""
    m = re.search(r"struct Options \{(.*?)\n\s*std::atomic<long long>\* find\(", text, flags=re.S)
    if not m:
        raise ValueError("struct Options / its find() not found")
    body = re.sub(r"//[^\n]*", "", m.group(1))
    defaults = {}
    for decl in re.findall(r"std::atomic<long long>\s+([^;]*);", body):
        d = re.fullmatch(r"\s*(\w+)\s*\{\s*(-?\d+)\s*\}\s*", decl)
        if not d:
            raise ValueError(f"option member without an integer default in its initialiser: {decl.strip()!r}")
        defaults[d.group(1)] = int(d.group(2))
    table = re.search(r"static const Entry table\[\] = \{(.*?)\};", text[m.end():], flags=re.S)
    if not table:
        raise ValueError("the find() table of struct Options not found")
    entries = re.findall(r'\{\s*"(\w+)"\s*,\s*&Options::(\w+)\s*\}', table.group(1))
    names = [name for name, _ in entries]
    if len(set(names)) != len(names):
        raise ValueError("an option name appears twice in the find() table")
    fields = {field for _, field in entries}
    if fields != set(defaults):
        raise ValueError(f"members missing from the find() table: {sorted(set(defaults) - fields)}; "
                         f"table entries without a member: {sorted(fields - set(defaults))}")
    return {name: defaults[field] for name, field in entries}


with open(HOST_H) as _f:
    DEFAULTS = parse_options(_f.read())


def snapshot() -> dict:
    return {k: pigo_b200.get_option(k) for k in DEFAULTS}


def _restore(values: dict):
    for k, v in values.items():
        if pigo_b200.get_option(k) != v:   # setting "timing" clears the timing counters: only write what changed
            pigo_b200.set_option(k, v)


@contextlib.contextmanager
def options(**overrides):
    """Runs the body with the given options set, then restores every option (also on an exception)."""
    unknown = sorted(set(overrides) - set(DEFAULTS))
    if unknown:
        raise KeyError(f"unknown options {unknown}")
    saved = snapshot()
    try:
        for k, v in overrides.items():
            pigo_b200.set_option(k, v)
        yield
    finally:
        _restore(saved)


@pytest.fixture(autouse=True)
def options_at_defaults():
    yield
    leaked = {k: v for k, v in snapshot().items() if v != DEFAULTS[k]}
    if leaked:
        _restore(DEFAULTS)
        pytest.fail("the test left options changed: " + ", ".join(f"{k}={v} (default {DEFAULTS[k]})" for k, v in sorted(leaked.items())),
                    pytrace=False)
