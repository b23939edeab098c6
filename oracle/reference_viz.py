"""Recipe that adds the reference's `viz_scripts/`, unmodified, to the Python install oracle/reference.py writes
(oracle/_ref/SplaTAM, git-ignored), so that tests can open a run record with the reference's own reader
(`viz_scripts/final_recon.py:load_camera`).  The source is oracle/reference.py's; where it cannot be read this is a
no-op."""
import os
import shutil

from . import reference

SUB = "viz_scripts"


def install():
    """Copies <source>/viz_scripts to oracle/_ref/SplaTAM/viz_scripts.  Returns True when the copy is in place."""
    src = reference.source_dir()
    if src is None or not os.path.isdir(os.path.join(src, SUB)):
        return False
    dst = os.path.join(reference.PY_DST, SUB)
    if os.path.isdir(dst):
        reference._make_writable(dst)
        shutil.rmtree(dst)
    shutil.copytree(os.path.join(src, SUB), dst)
    reference._make_writable(dst)           # the source modes may be read-only; keep the install removable
    return True


if __name__ == "__main__":
    print("reference viz_scripts in oracle/_ref:", install())
