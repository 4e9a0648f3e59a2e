"""The learner's prune_rare key on the host (no GPU): parsing, the checkpoint fingerprint that records it only when it
is set, and the refusal by name of a resume under another value (difacto_b200/host/tests/prune_rare_settings_tests.cc)."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_prune_rare_key_and_the_checkpoint_fingerprint():
    sys.path.insert(0, ROOT)
    from difacto_b200 import build as eb
    from difacto_b200.host import build as hb
    eb.build()
    out = subprocess.run([os.path.join(hb.build(), "prune_rare_settings_tests")], capture_output=True, text=True)
    assert out.returncode == 0 and out.stdout.strip() == "ok", out.stdout + out.stderr
