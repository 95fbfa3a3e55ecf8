"""CPU: every script in tools/ compiles, and every absolute import in it resolves, so a refactor of the package cannot
leave a benchmark that fails only when someone next runs it on a GPU."""
import ast
import glob
import importlib
import importlib.util
import os
import py_compile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOOLS = os.path.join(ROOT, "tools")


def _imports(path):
    """(line, module, names) of every absolute import in the file, inside functions too; names is None for `import X`."""
    for node in ast.walk(ast.parse(open(path).read(), path)):
        if isinstance(node, ast.Import):
            for a in node.names:
                yield node.lineno, a.name, None
        elif isinstance(node, ast.ImportFrom) and node.level == 0:
            yield node.lineno, node.module, [a.name for a in node.names]


@pytest.mark.parametrize("name", sorted(os.path.basename(p) for p in glob.glob(os.path.join(TOOLS, "*.py"))))
def test_tool_compiles_and_its_imports_resolve(name, tmp_path, monkeypatch):
    path = os.path.join(TOOLS, name)
    py_compile.compile(path, cfile=str(tmp_path / "tool.pyc"), doraise=True)
    for p in (os.path.join(ROOT, "tests"), os.path.join(ROOT, "dinov3-jax_b200"), ROOT, TOOLS):     # bench_convnext reads tests/
        monkeypatch.syspath_prepend(p)
    missing = []
    for line, module, names in _imports(path):
        try:
            mod = importlib.import_module(module)
        except ImportError as e:
            missing.append(f"{name}:{line}: {module} ({e})")
            continue
        for n in names or ():
            if not hasattr(mod, n) and not (hasattr(mod, "__path__") and importlib.util.find_spec(f"{module}.{n}")):
                missing.append(f"{name}:{line}: {n} from {module}")
    assert not missing, missing
