"""Recipe for oracle/_ref/: the unmodified facebookresearch/esm package, used by the drop-in tests and by bench.py's
reference legs.  The package is pure Python, so "building" it is copying its `esm/` directory out of a source checkout
given by ESM_REFERENCE_SRC (default: /root/reference).  oracle/_ref/ is git-ignored; once made, it travels with the
tree to machines that have no reference checkout, and a later build() there leaves it as it is."""
import os
import shutil

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_DIR = os.path.join(ROOT, "oracle", "_ref")


def build(src: str | None = None) -> bool:
    """Copy <src>/esm to oracle/_ref/esm; returns whether oracle/_ref/esm is present afterwards."""
    src = src or os.environ.get("ESM_REFERENCE_SRC", "/root/reference")
    pkg = os.path.join(src, "esm")
    if os.path.isfile(os.path.join(pkg, "__init__.py")):
        tmp = REF_DIR + ".tmp"
        shutil.rmtree(tmp, ignore_errors=True)
        shutil.copytree(pkg, os.path.join(tmp, "esm"), ignore=shutil.ignore_patterns("__pycache__", "*.pyc"))
        for dp, dns, fns in os.walk(tmp):  # files copied from a read-only tree are read-only: make the copy replaceable
            for n in dns:
                os.chmod(os.path.join(dp, n), 0o755)
            for n in fns:
                os.chmod(os.path.join(dp, n), 0o644)
        shutil.rmtree(REF_DIR, ignore_errors=True)
        os.replace(tmp, REF_DIR)
    return os.path.isdir(os.path.join(REF_DIR, "esm"))
