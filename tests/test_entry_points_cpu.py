"""The entry-point ledger (tests/entry_points.py) against the header and the package's sources: every declared symbol
is owned or listed as not launched, never both; each owner file names the symbols it owns (or their lib wrappers);
and the package reaches the shared library only through lib.call, so that patching lib.call sees every launch."""
import ast
import glob
import os
import re
import sys

sys.path.insert(0, os.path.dirname(__file__))
import entry_points as E  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "open-musiclm_b200")
TESTS = os.path.dirname(os.path.abspath(__file__))


def _lib():
    from open_musiclm_b200 import lib
    return lib


def wrappers():
    """symbol -> the top-level functions and classes of lib.py whose bodies name it."""
    tree = ast.parse(open(os.path.join(PKG, "lib.py")).read())
    out = {}
    for node in tree.body:
        if isinstance(node, (ast.FunctionDef, ast.ClassDef)):
            for c in ast.walk(node):
                if isinstance(c, ast.Constant) and isinstance(c.value, str) and c.value.startswith("omlm_"):
                    out.setdefault(c.value, set()).add(node.name)
    return out


def test_ledger_covers_the_header_exactly():
    owned, dead = set(E.OWNER), set(E.NOT_LAUNCHED)
    assert not owned & dead, f"both owned and not launched: {sorted(owned & dead)}"
    header = set(_lib().header_symbols())
    assert owned | dead == header, \
        f"declared but not in the ledger: {sorted(header - owned - dead)}; in the ledger but not declared: {sorted(owned | dead - header)}"
    assert set(E.OUTSIDE_PHASES) <= owned and E.DIRECT_HOST_CALLS <= {s for s, o in E.OWNER.items() if o == E.HOST}
    assert all(r.strip() for r in E.NOT_LAUNCHED.values()) and all(r.strip() for r in E.OUTSIDE_PHASES.values())


def test_every_owner_file_names_its_symbols():
    """A text check: the owner file names the symbol (with or without omlm_), or a lib wrapper that launches at most
    two symbols (a flag picks the variant: det, ragged, invariant).  lib.sample, which picks among five, does not count."""
    wrap = wrappers()
    fanout = {}
    for s, ws in wrap.items():
        for w in ws:
            fanout[w] = fanout.get(w, 0) + 1
    missing = []
    for sym, owner in sorted(E.OWNER.items()):
        if owner == E.HOST:
            continue
        path = os.path.join(TESTS, owner)
        assert os.path.exists(path), f"{sym}: owner file {owner} does not exist"
        src = open(path).read()
        names = {sym, sym[len("omlm_"):]} | {w for w in wrap.get(sym, set()) if fanout[w] <= 2}
        if not any(re.search(rf"\b{re.escape(n)}\b", src) for n in names):
            missing.append(f"{sym} ({owner}: none of {sorted(names)})")
    assert not missing, f"owner files that do not name their symbols: {missing}"


def _direct_calls(path):
    """(line, what) of every way a module reaches the CDLL other than lib.call: ctypes.CDLL, getattr on load(), and
    attributes of load(), lib.load() or lib._lib."""
    tree = ast.parse(open(path).read())
    is_lib = os.path.basename(path) == "lib.py"
    found = []
    funcs = {}
    for node in ast.walk(tree):
        if isinstance(node, ast.FunctionDef):
            for c in ast.walk(node):
                funcs.setdefault(id(c), node.name)

    def is_handle(v):
        if isinstance(v, ast.Call) and isinstance(v.func, ast.Name) and v.func.id == "load":
            return True
        if isinstance(v, ast.Call) and isinstance(v.func, ast.Attribute) and v.func.attr == "load":
            return True
        return (isinstance(v, ast.Name) and v.id == "_lib" and is_lib) or (isinstance(v, ast.Attribute) and v.attr == "_lib")

    for node in ast.walk(tree):
        fn = funcs.get(id(node))
        if isinstance(node, ast.Attribute) and node.attr == "CDLL" and not (is_lib and fn == "load"):
            found.append((node.lineno, "ctypes.CDLL"))
        if isinstance(node, ast.Call) and isinstance(node.func, ast.Name) and node.func.id == "getattr" and node.args and \
                is_handle(node.args[0]) and not (is_lib and fn == "call"):
            found.append((node.lineno, "getattr on the library handle"))
        if isinstance(node, ast.Attribute) and is_handle(node.value) and node.attr not in E.DIRECT_HOST_CALLS:
            found.append((node.lineno, node.attr))
    return found


def test_the_package_launches_only_through_lib_call():
    bad = []
    for path in sorted(glob.glob(os.path.join(PKG, "*.py"))):
        bad += [f"{os.path.basename(path)}:{line}: {what}" for line, what in _direct_calls(path)]
    assert not bad, f"calls into the shared library that bypass lib.call: {bad}"


def test_the_direct_call_check_sees_a_bypass(tmp_path):
    """The scan flags a module that calls an entry point on load() or through getattr, and passes lib.py's own two."""
    p = tmp_path / "mod.py"
    p.write_text("from . import lib\n\ndef f():\n    lib.load().omlm_sample(1)\n    getattr(lib.load(), 'omlm_pack')()\n")
    assert [w for _, w in _direct_calls(str(p))] == ["omlm_sample", "getattr on the library handle"]
    assert _direct_calls(os.path.join(PKG, "lib.py")) == []
