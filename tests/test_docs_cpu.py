"""Keeps the documentation honest: every test, source file and profile the docs point at must exist."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DOCS = ["README.md", "DESIGN.md", "docs/MIGRATING.md"]


def _read(rel):
    with open(os.path.join(ROOT, rel)) as f:
        return f.read()


def _all_test_names():
    names = set()
    for fn in os.listdir(os.path.join(ROOT, "tests")):
        if fn.startswith("test_") and fn.endswith(".py"):
            names.update(re.findall(r"^def (test_\w+)", _read(os.path.join("tests", fn)), flags=re.M))
    return names


def test_tests_named_in_the_docs_exist():
    have = _all_test_names()
    missing = []
    for doc in DOCS:
        for name in set(re.findall(r"\b(test_[a-z0-9_]+)\b", _read(doc))):
            if name.endswith("_cpu") or name.endswith("_gpu") or os.path.exists(os.path.join(ROOT, "tests", name + ".py")):
                continue                                   # a test *file* name
            if name.endswith("_"):                         # prefix wildcard such as test_logger_*
                if not any(h.startswith(name) for h in have):
                    missing.append((doc, name))
            elif name not in have and not any(h.startswith(name) for h in have):
                missing.append((doc, name))
    assert not missing, missing


def test_paths_named_in_the_docs_exist():
    missing = []
    for doc in DOCS:
        base = os.path.dirname(doc)
        for path in set(re.findall(r"`((?:b200ddp|csrc|tests|tools|bench|docs|profiles|baseline)/[\w./-]+?\.(?:py|cu|cuh|cpp|h|md|sh|json|txt))`", _read(doc))):
            cands = [path, os.path.join("b200ddp", path), os.path.join(base, path)]
            if not any(os.path.exists(os.path.join(ROOT, c)) for c in cands):
                missing.append((doc, path))
    assert not missing, missing
