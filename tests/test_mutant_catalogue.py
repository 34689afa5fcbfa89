"""The mutant catalogue of tools/mutants.py stays applicable: every snippet still occurs exactly once in its file, every
mapped test file exists, and every mutant marked equivalent names a proof test that exists.  Cheap: nothing is built."""
import ast
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import mutants  # noqa: E402


def test_every_snippet_occurs_exactly_once():
    stale = [(e["id"], mutants.snippet_count(e)) for e in mutants.CATALOGUE if mutants.snippet_count(e) != 1]
    assert not stale, stale


def test_entries_are_well_formed():
    ids = [e["id"] for e in mutants.CATALOGUE]
    assert len(ids) == len(set(ids))
    for e in mutants.CATALOGUE:
        assert e["find"] != e["repl"], e["id"]
        assert e["tests"], e["id"]
        for t in e["tests"]:
            assert os.path.isfile(os.path.join(ROOT, t)), (e["id"], t)


def test_equivalent_mutants_name_an_existing_proof():
    for e in mutants.CATALOGUE:
        if not e["equivalent"]:
            assert e["proof"] is None, e["id"]
            continue
        path, name = e["proof"].split("::")
        with open(os.path.join(ROOT, path)) as f:
            tree = ast.parse(f.read())
        assert name in {n.name for n in tree.body if isinstance(n, ast.FunctionDef)}, e["id"]
