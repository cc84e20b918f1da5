"""Install the UNMODIFIED reference under oracle/_ref/, next to the oracle that imports it.

microsoft/esvit has no setup.py / pyproject (SURVEY.md section 0), so `pip install --target oracle/_ref
<reference checkout>` has nothing to build; "installing" it is a verbatim copy of its Python sources and experiment YAMLs.
oracle/_ref/ is git-ignored (it never enters the history - the repo holds no reference source) and travels with the
built tree, so bench.py's reference arms import the reference's own modules from it on the GPU machine:
`bench.py --impl reference --device cuda` and the `gpu_reference` entry of the default bench line.

Run by __graft_entry__.build() when the reference checkout (ESVIT_REFERENCE_SRC, default /root/reference) is readable;
a no-op without one, so a tree that already holds oracle/_ref/ keeps it."""
from __future__ import annotations

import os
import shutil
import sys

SRC = os.environ.get("ESVIT_REFERENCE_SRC", "/root/reference")
DST = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref")
KEEP_EXT = (".py", ".yaml", ".yml", ".txt", ".md")


def install(force: bool = False) -> str:
    if not os.path.isfile(os.path.join(SRC, "main_esvit.py")):
        return DST if os.path.isdir(DST) else ""
    stamp = os.path.join(DST, ".installed")
    if os.path.isfile(stamp) and not force:
        return DST
    if os.path.isdir(DST):
        shutil.rmtree(DST)
    for root, dirs, files in os.walk(SRC):
        dirs[:] = [d for d in dirs if d not in (".git", "__pycache__", "plot")]
        rel = os.path.relpath(root, SRC)
        for f in files:
            if f.endswith(KEEP_EXT):
                os.makedirs(os.path.join(DST, rel), exist_ok=True)
                shutil.copy2(os.path.join(root, f), os.path.join(DST, rel, f))
    open(stamp, "w").write("copied verbatim from %s\n" % SRC)
    return DST


if __name__ == "__main__":
    print(install(force="--force" in sys.argv))
