"""The learner's prune_period / prune_count keys on the host (no GPU): parsing, their checks, and the checkpoint
fingerprint that refuses a resume under other prune settings by name (difacto_b200/host/tests/prune_settings_tests.cc)."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_prune_keys_and_the_checkpoint_fingerprint():
    sys.path.insert(0, ROOT)
    from difacto_b200 import build as eb
    from difacto_b200.host import build as hb
    eb.build()
    out = subprocess.run([os.path.join(hb.build(), "prune_settings_tests")], capture_output=True, text=True)
    assert out.returncode == 0 and out.stdout.strip() == "ok", out.stdout + out.stderr
