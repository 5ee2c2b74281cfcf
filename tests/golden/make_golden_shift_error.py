"""Writes ref_shift_error.json: the relative errors the reference's own test_shifted.c, built with -DDISPLAY_ERROR on its own sources
(oracle/_ref/ref_test_shifted_error_stock, oracle/shift_error.mk), prints for its five shifts on test_shifted_convdiff16.mtx
(test_shifted.c:129-154).  The stored values are that program's output, not its code.

    python tests/golden/make_golden_shift_error.py"""
import json
import os
import re
import subprocess
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
LINE = re.compile(r"^(#seed|sigma): (\S+), relative error: (\S+)$", re.M)


def parse(stdout):
    """[(is_seed, sigma, relative error)] of test_shifted.c's DISPLAY_ERROR lines, in print order."""
    return [(m.group(1) == "#seed", float(m.group(2)), float(m.group(3))) for m in LINE.finditer(stdout)]


def main():
    exe = os.path.join(ROOT, "oracle", "_ref", "ref_test_shifted_error_stock")
    mtx = os.path.join(HERE, "test_shifted_convdiff16.mtx")
    with tempfile.TemporaryDirectory() as d:
        p = subprocess.run([exe, mtx], capture_output=True, text=True, check=True, cwd=d)
    rows = parse(p.stdout)
    assert len(rows) == 5, p.stdout
    total_iter = int(re.search(r"Total iter\s*:\s*(\d+)", p.stdout).group(1))
    out = {"mtx": os.path.basename(mtx), "total_iter": total_iter,
           "lines": [{"seed": s, "sigma": sg, "relative_error": e} for s, sg, e in rows]}
    with open(os.path.join(HERE, "ref_shift_error.json"), "w") as f:
        json.dump(out, f, indent=1)
        f.write("\n")
    print(out)


if __name__ == "__main__":
    main()
