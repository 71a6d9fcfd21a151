"""TEST / BASELINE INFRASTRUCTURE ONLY — recipe that places the reference's own SVA implementation under oracle/_ref/.

    python oracle/make_ref.py          (run by __graft_entry__.build() when /root/reference exists)

The reference is pure Python; the one file of its hot path that needs nothing but torch is
`cambrian/model/vision_sampler.py` (VisionTokenSampler, vision_sampler.py:407-419).  It is copied VERBATIM, byte for
byte, from where it lies under /root/reference into oracle/_ref/ — a git-ignored build OUTPUT, like the built .so — so
that the CPU arm of bench.py (oracle/cpu_arm.py) can time the reference's real module on machines where the reference
tree does not exist.  Nothing under oracle/_ref/ is committed, imported by the product, or edited.
"""
from __future__ import annotations

import hashlib
import os
import shutil

SRC = "/root/reference/cambrian/model/vision_sampler.py"
DST_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref")


def make() -> str | None:
    if not os.path.exists(SRC):
        return None
    os.makedirs(DST_DIR, exist_ok=True)
    dst = os.path.join(DST_DIR, "vision_sampler.py")
    shutil.copyfile(SRC, dst)
    digest = hashlib.sha256(open(dst, "rb").read()).hexdigest()
    with open(os.path.join(DST_DIR, "SOURCE.txt"), "w") as f:
        f.write(f"{SRC}\nsha256 {digest}\ncopied verbatim by oracle/make_ref.py; do not edit, do not commit\n")
    return dst


if __name__ == "__main__":
    print(make() or "reference tree not present: nothing to do")
