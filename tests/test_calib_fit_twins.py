"""k_calib_fit and k_calib_fit_w (distributed_sgd_b200/csrc/dsgd_calibrate.cuh) are one fit written twice, so that the
unweighted kernel keeps its instructions: the weighted one must differ only in its weighted lines.  CPU only."""
import difflib
import os
import re

SRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "distributed_sgd_b200", "csrc",
                   "dsgd_calibrate.cuh")


def body(src, name):
    start = src.index(f"k_calib_{name}(const CalibFitParams p) {{")
    depth, i = 0, src.index("{", start)
    for j in range(i, len(src)):
        depth += {"{": 1, "}": -1}.get(src[j], 0)
        if depth == 0:
            return src[i:j + 1].splitlines()


def test_the_weighted_fit_differs_only_in_its_weighted_lines():
    src = open(SRC).read()
    a, b = body(src, "fit"), body(src, "fit_w")
    changed = [l[1:].strip() for l in difflib.unified_diff(a, b, lineterm="", n=0)
               if l[:1] in "+-" and not l.startswith(("+++", "---"))]
    allowed = re.compile(r"s_c|p\.cw|\bc \* |c\[|rint\(c \* 0x1p160\)|cal_add\(lim\[\d\], ovf, (term|f \* d1|d1|\(f \* f\) \* d2|"
                         r"f \* d2|d2)\);|int8_t \*s_y")
    assert changed, "the two kernels are identical: the weighted lines are missing"
    assert all(allowed.search(l) for l in changed), [l for l in changed if not allowed.search(l)]
