"""Generate tests/golden/ref_driver_test_shifted.json: the external symbols of the reference's unchanged test_shifted.c (the driver
of shifted_solver.c) compiled against include/compat/mpi.h -- what a program built from it needs the library (and libc / libm)
to provide.  Same procedure as make_golden_drivers.py for the other drivers.  Run with a checkout of the reference:
    BICG_REFERENCE_DIR=<checkout> python tests/golden/make_golden_driver_test_shifted.py
"""
import json
import os
import subprocess
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
SRC = os.path.join(os.environ["BICG_REFERENCE_DIR"], "src")

with tempfile.TemporaryDirectory() as td:
    obj = os.path.join(td, "test_shifted.o")
    subprocess.run(["gcc", "-O2", "-w", "-I" + os.path.join(ROOT, "include", "compat"), "-I" + SRC, "-c",
                    os.path.join(SRC, "test_shifted.c"), "-o", obj], check=True)
    nm = subprocess.run(["nm", "-u", obj], capture_output=True, text=True, check=True).stdout
    syms = sorted(l.split()[-1] for l in nm.splitlines() if l.strip())
    print("test_shifted.c", len(syms), "undefined symbols")
with open(os.path.join(ROOT, "tests", "golden", "ref_driver_test_shifted.json"), "w") as f:
    json.dump({"test_shifted.c": syms}, f, indent=1)
    f.write("\n")
