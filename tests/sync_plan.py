"""Runs the batched sync calls' host planner (csrc/sync_plan.h, plan_sync) on the CPU through
tests/host_emul/plan_emul: the argument checks, the reference / chunk / tokenizer tables and the sub-batch cuts
the b2_sync_* entry points compute before they launch anything."""
import os
import subprocess
import tempfile

import numpy as np

from conftest import ROOT

EMUL = os.path.join(ROOT, "tests", "host_emul", "plan_emul")


def plan(**req):
    """req: the fields plan_emul.cu reads (arrays as sequences, None = null pointer).  Returns a dict with
    "status", "err" and every table of the plan as an int64 array."""
    if not os.path.exists(EMUL):
        import sys
        sys.path.insert(0, ROOT)
        import __graft_entry__ as ge
        ge.build()
    with tempfile.TemporaryDirectory() as d:
        src, dst = os.path.join(d, "in.txt"), os.path.join(d, "out.txt")
        with open(src, "w") as f:
            for k, v in req.items():
                if v is None:
                    continue
                vals = [v] if np.isscalar(v) or isinstance(v, str) else list(np.asarray(v).ravel())
                f.write("%s %d %s\n" % (k, len(vals), " ".join(repr(float(x)) if isinstance(x, (float, np.floating))
                                                              else str(int(x)) if not isinstance(x, str) else x
                                                              for x in vals)))
        subprocess.check_call([EMUL, src, dst])
        out = {}
        for line in open(dst).read().splitlines():
            k, _, rest = line.partition(" ")
            if k == "status":
                out[k] = int(rest)
            elif k == "err":
                out[k] = rest
            elif k == "two_level":
                a, b = rest.split()
                out[k], out["ref_label"] = bool(int(a)), float(b)
            else:
                out[k] = np.array([int(x) for x in rest.split()], dtype=np.int64)
        return out
