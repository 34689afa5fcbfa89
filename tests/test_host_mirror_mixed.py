"""Commits of a mixed ECDSA / Ed25519 consenter set from the wire in the C++ host mirror (consensus_b200/host/marshal.hpp,
CommitBatch::Mixed): TestMixedCommitBatch of host_tests.  Without a GPU it checks the decoding and registration rules
(which wire Commits are inert, which are registered with a rejecting row, and the scheme, slot and signature row of the
others); on the GPU one sbv_mixed_verify_quorum call is compared vote by vote with the reference's VoteSet rule."""
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST = os.path.join(ROOT, "consensus_b200", "host")


def _run(mode, timeout):
    subprocess.check_call(["make", "-s", "-C", HOST, "host_tests"])
    out = subprocess.run([os.path.join(HOST, "host_tests"), mode], capture_output=True, text=True, timeout=timeout)
    assert out.returncode == 0, out.stdout + out.stderr
    assert re.search(r"^TestMixedCommitBatch\s+ok$", out.stdout, re.M), out.stdout + out.stderr
    assert " 0 failures" in out.stdout


def test_mixed_commit_decoding_rules():
    _run("cpu", 120)


@pytest.mark.gpu
def test_mixed_commit_batch_on_the_engine():
    _run("gpu", 300)
