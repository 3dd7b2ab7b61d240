#!/usr/bin/env python
"""Recipe for `oracle/_ref/`: the reference's own hot-path modules, BYTE-COMPILED from the sources of a reference
checkout (D4PG_REFERENCE_PATH; no source is copied into this repository; `oracle/_ref/` is git-ignored build output,
like the built .so files).

    python oracle/build_ref.py          # run by __graft_entry__.build() whenever the reference checkout exists

The seven modules are the ones `oracle/ref_shim.py` imports: ddpg.py (DDPG.train, ddpg.py:200-255),
prioritized_replay_memory.py, replay_memory.py, models.py, shared_adam.py, utils.py, random_process.py.  They are
pure Python, so "building" them is `py_compile` to sourceless `<name>.pyc` files, importable by the same CPython
version (3.12).  `bench.py --impl reference` and the `cpu_baseline` leg then time the UNMODIFIED
reference (`cpu_baseline.kind = "reference"`) behind the 4-item shim of ref_shim.py; without `oracle/_ref/` they
fall back to the oracle port (`kind = "port"`).  TEST / BENCH INFRASTRUCTURE ONLY -- never imported by the product.
"""
import os
import py_compile
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "_ref")
SRC = os.environ.get("D4PG_REFERENCE_PATH", "/root/reference")
MODULES = ["utils", "models", "random_process", "replay_memory", "prioritized_replay_memory", "shared_adam", "ddpg"]


def build(verbose=False):
    """Returns the output directory, or None when the reference sources are not present (then a previously built oracle/_ref/ is used as it is)."""
    if not os.path.isfile(os.path.join(SRC, "ddpg.py")):
        return OUT if os.path.isfile(os.path.join(OUT, "ddpg.pyc")) else None
    os.makedirs(OUT, exist_ok=True)
    for m in MODULES:
        src, dst = os.path.join(SRC, m + ".py"), os.path.join(OUT, m + ".pyc")
        # unchecked-hash pycs: valid without the source file next to them
        py_compile.compile(src, cfile=dst, dfile="reference/%s.py" % m, doraise=True,
                           invalidation_mode=py_compile.PycInvalidationMode.UNCHECKED_HASH)
        if verbose:
            print("compiled %s -> %s" % (src, dst))
    with open(os.path.join(OUT, "PROVENANCE"), "w") as f:
        f.write("byte-compiled from %s by oracle/build_ref.py with CPython %s; no sources copied\n" % (SRC, sys.version.split()[0]))
    return OUT


if __name__ == "__main__":
    print(build(verbose=True))
