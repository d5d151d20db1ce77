"""Stage the UNMODIFIED reference under oracle/_ref/ (git-ignored; build() runs this, so the staged copy travels with
a built tree to machines that have no reference checkout).

The reference (SHI-Labs/Prompt-Free-Diffusion) is an un-packaged Python app: no setup.py / pyproject, it runs
only from its own checkout with `lib/` and `configs/` resolved relative to the CWD (lib/cfg_helper.py:104), so
`pip install --target oracle/_ref <reference>` has nothing to build (DESIGN.md §6).  The install step is
therefore a verbatim copy of the two directories the model_zoo needs (0.8 MB; assets/ and app.py are not needed:
app.py cannot be imported without gradio / pretrained weights).  Nothing under oracle/_ref is ever edited,
imported by the product, or committed.

    python oracle/install_reference.py     # keeps an existing oracle/_ref when no reference checkout is found
"""
import os
import shutil
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.environ.get("PFD_REFERENCE_SRC", "/root/reference")
DST = os.path.join(ROOT, "oracle", "_ref")


def install(verbose=True) -> bool:
    if not os.path.isdir(os.path.join(SRC, "lib", "model_zoo")):
        if verbose:
            print(f"[install_reference] {SRC} not present: keeping whatever is in {DST}")
        return os.path.isdir(os.path.join(DST, "lib", "model_zoo"))
    for sub in ("lib", "configs"):
        d = os.path.join(DST, sub)
        if os.path.isdir(d):
            shutil.rmtree(d)
        shutil.copytree(os.path.join(SRC, sub), d, ignore=shutil.ignore_patterns("__pycache__", "*.pyc"))
    for f in ("LICENSE", "README.md", "requirements.txt"):
        if os.path.exists(os.path.join(SRC, f)):
            shutil.copy2(os.path.join(SRC, f), os.path.join(DST, f))
    if verbose:
        print(f"[install_reference] copied lib/ and configs/ of {SRC} to {DST}")
    return True


if __name__ == "__main__":
    sys.exit(0 if install() else 1)
