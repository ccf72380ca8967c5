"""The entry-point ledger (tests/entry_points.py) against what the engine really launches: lib.call patched over every
phase of every model of tests/call_forms.py, in both act16 modes.  Every launched symbol must be owned, no symbol
listed as not launched may be launched, and every owned symbol must be launched in some phase (host queries that lib
calls directly and the symbols of OUTSIDE_PHASES aside), so the ledger cannot go stale in either direction."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(__file__))
import call_forms  # noqa: E402
import entry_points as E  # noqa: E402

pytestmark = pytest.mark.gpu


class _Launches:
    """Patches lib.call (every wrapper looks it up as a module global at call time) and files each symbol under the
    current phase.  Host-only: no device memory is read."""

    def __init__(self, lib):
        self.lib, self.orig, self.phase, self.seen = lib, lib.call, None, {}

    def __enter__(self):
        def call(name, *args):
            self.seen.setdefault(name, set()).add(self.phase)
            return self.orig(name, *args)
        self.lib.call = call
        return self

    def __exit__(self, *exc):
        self.lib.call = self.orig


def test_launched_symbols_match_the_ledger(monkeypatch):
    from open_musiclm_b200 import lib
    with _Launches(lib) as rec:
        for act16 in ("bf16", "fp16"):
            for model in call_forms.MODEL_KEYS:
                call_forms.run(_Phase(rec, f"{model} {act16}"), model, act16, monkeypatch)
    seen = rec.seen
    unowned = sorted(f"{s} (in {sorted(p)[:3]})" for s, p in seen.items() if s not in E.OWNER and s not in E.NOT_LAUNCHED)
    dead = sorted(f"{s} (in {sorted(p)[:3]})" for s, p in seen.items() if s in E.NOT_LAUNCHED)
    exempt = E.DIRECT_HOST_CALLS | set(E.OUTSIDE_PHASES)
    stale = sorted(s for s in E.OWNER if s not in seen and s not in exempt)
    print("launched:", {s: len(p) for s, p in sorted(seen.items())})
    assert not unowned, f"launched symbols without an owner in entry_points.OWNER: {unowned}"
    assert not dead, f"symbols listed in entry_points.NOT_LAUNCHED that the engine launched: {dead}"
    assert not stale, f"owned symbols no phase launched (move them to NOT_LAUNCHED, or add the phase): {stale}"


class _Phase:
    """A recorder for call_forms.run that prefixes each phase with the model and act16 mode before handing it on."""

    def __init__(self, rec, tag):
        self.rec, self.tag = rec, tag

    @property
    def phase(self):
        return self.rec.phase

    @phase.setter
    def phase(self, p):
        self.rec.phase = f"{self.tag}: {p}"
