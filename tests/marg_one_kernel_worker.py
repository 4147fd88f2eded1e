"""Worker of tests/test_marginalize_edges.py::test_one_kernel_eigen_path: libviwb reads VIWB_MARG_ONE_KERNEL when it loads, so the one-kernel
eigen path (marg_eig) runs in a process of its own.  Marginalises the cases of path_cases() and writes every prior to an .npz.
Usage: marg_one_kernel_worker.py <library path, empty for the product library> <output .npz>"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "viw-fusion_b200", "python"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402

import test_marginalize_edges as edges  # noqa: E402
import viw_oracle  # noqa: E402
from viwb import lib  # noqa: E402

viw_oracle.lib()
ctx = lib.Context(0, sys.argv[1] or None)
out = {}
for name, (p, a, flag) in edges.path_cases(viw_oracle).items():
    out.update(ctx.marginalize(p, a, flag).to_npz_dict(name + "."))
np.savez(sys.argv[2], **out)
ctx.close()
