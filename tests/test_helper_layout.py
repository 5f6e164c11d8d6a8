"""Test modules import helpers, never each other (DESIGN §5b): no module under tests/ or tools/ imports a module whose
name starts with test_, and none imports a name `env` (each GPU module declares its own module fixture)."""
import ast
import glob
import os

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _imports(path):
    """(line, imported module, imported names) of every import statement in the file."""
    for node in ast.walk(ast.parse(open(path).read(), path)):
        if isinstance(node, ast.Import):
            for a in node.names:
                yield node.lineno, a.name, ()
        elif isinstance(node, ast.ImportFrom) and node.module:
            yield node.lineno, node.module, tuple(a.name for a in node.names)


def test_no_module_imports_a_test_module_or_a_fixture():
    files = sorted(glob.glob(os.path.join(ROOT, "tests", "**", "*.py"), recursive=True) +
                   glob.glob(os.path.join(ROOT, "tools", "**", "*.py"), recursive=True))
    assert files
    bad = []
    for f in files:
        for line, module, names in _imports(f):
            if module.split(".")[-1].startswith("test_") or any(n.startswith("test_") for n in names) \
                    or "env" in names:
                bad.append("%s:%d imports %s %s" % (os.path.relpath(f, ROOT), line, module, ", ".join(names)))
    assert not bad, "\n".join(bad)
