"""Compile the UNMODIFIED reference into oracle/_ref/ as bytecode.  TEST INFRASTRUCTURE.

    python -m oracle.build_ref        (also run by __graft_entry__.build() where the reference is readable)

The reference's Python packages (`trajnetbaselines`, `evaluator`) are compiled module by module into sourceless
`.pyc` files (no `.py` is copied), and its `DATA_BLOCK` ndjson data is copied beside them, so that
`oracle/ref_shim.py` can import the reference on a machine that has only this tree: the drop-in tests
(tests/test_dropin.py), the live oracle checks (tests/test_oracle_vs_reference.py), the `DATA_BLOCK` parser tests and
`bench.py --impl reference`.  oracle/_ref/ is a build product (git-ignored).
"""
import os
import py_compile
import shutil
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "_ref")
PACKAGES = ("trajnetbaselines", "evaluator")


def source_root():
    root = os.environ.get("TRAJNET_REFERENCE_SRC", "/root/reference")
    return root if os.access(os.path.join(root, "trajnetbaselines", "__init__.py"), os.R_OK) else None


def build(force=False):
    """Returns OUT, or None when the reference sources are not readable here."""
    src = source_root()
    if src is None:
        return None
    stamp = os.path.join(OUT, ".complete")
    if os.path.exists(stamp) and not force:
        return OUT
    tmp = OUT + ".tmp"
    shutil.rmtree(tmp, ignore_errors=True)
    for pkg in PACKAGES:
        for dirpath, dirnames, filenames in os.walk(os.path.join(src, pkg)):
            dirnames[:] = [d for d in dirnames if d != "__pycache__"]
            rel = os.path.relpath(dirpath, src)
            for fn in filenames:
                if fn.endswith(".py"):
                    dst = os.path.join(tmp, rel, fn[:-3] + ".pyc")
                    os.makedirs(os.path.dirname(dst), exist_ok=True)
                    py_compile.compile(os.path.join(dirpath, fn), cfile=dst, dfile=os.path.join(rel, fn), doraise=True,
                                       invalidation_mode=py_compile.PycInvalidationMode.UNCHECKED_HASH)
    shutil.copytree(os.path.join(src, "DATA_BLOCK"), os.path.join(tmp, "DATA_BLOCK"),
                    ignore=shutil.ignore_patterns("*.py", "*.pyc"))
    shutil.rmtree(OUT, ignore_errors=True)
    os.rename(tmp, OUT)
    open(stamp, "w").close()
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv))
