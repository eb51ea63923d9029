"""Record joint_oracle_sha1.json from the per-type joint oracles that tests/joint_oracle.c replaced.

    python tests/golden/make_joint_oracle_golden.py --root <checkout of the parent commit>

The parent commit (b49fa3e) defined each joint type the reference lacks by an oracle of its own, tests/<type>_oracle.c,
each loaded by tests/<type>_oracle.py. This script imports those loaders from --root and the worlds of
tests/test_joint_oracle_cpu.py from this tree, and records, for every world and variant, one truncated sha1 of the body
and joint rows of every step from the oracle the world names. Its revolute and mouse world is recorded from --root's
oracle/s2o_solver.c, built with the oracle's flags.
"""
import argparse
import hashlib
import importlib
import json
import os
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
TESTS = os.path.dirname(HERE)


def _base_oracle(root, port):
    out = os.path.join(tempfile.mkdtemp(), "libs2oracle_base.so")
    subprocess.run(["gcc", "-std=gnu17", "-O2", "-fPIC", "-fvisibility=default", "-Wall", "-I" + os.path.join(root, "include"),
                    "-shared", "-o", out, os.path.join(root, "oracle", "s2o_solver.c"), "-lm"], check=True)
    return port.Oracle(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--root", required=True, help="a checkout of the commit whose per-type oracles are recorded")
    root = os.path.abspath(ap.parse_args().root)
    # the parent's loaders first: they read ROOT from the parent's tests/helpers.py
    sys.path[:0] = [os.path.join(root, "tests"), root]
    from oracle import port
    names = ["weld", "soft_weld", "motor", "prismatic", "spring", "distance", "wheel", "pulley", "gear"]
    oracles = {name: importlib.import_module(f"{name}_oracle").load() for name in names}
    oracles["base"] = _base_oracle(root, port)
    sys.path.insert(0, TESTS)
    import test_joint_oracle_cpu as T

    worlds = {}
    for name, (build, steps, source) in T.WORLDS.items():
        worlds[name] = {solver: T.run_digest(oracles[source], solver, build, steps) for solver in T.VARIANTS}
    parent = subprocess.run(["git", "-C", root, "rev-parse", "HEAD"], check=True, capture_output=True, text=True).stdout.strip()
    path = os.path.join(HERE, "joint_oracle_sha1.json")
    with open(path, "w") as f:
        f.write('{\n"parent": %s,\n"worlds": {\n' % json.dumps(parent))
        f.write(",\n".join("%s: %s" % (json.dumps(w), json.dumps(v)) for w, v in worlds.items()))
        f.write("\n}\n}\n")
    print("wrote", path, hashlib.sha1(open(path, "rb").read()).hexdigest()[:16])


if __name__ == "__main__":
    main()
