"""The C++ host-layer test programs in tests/cpp: the problem file they read (tests/cpp/host_input.hpp) and the one
recipe they are compiled by."""
import os
import subprocess

import numpy as np

from trajopt_b200 import capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "trajopt_b200", "csrc")
_built = {}


def build(tmp_path_factory, name, shared=False, extra=()):
    """Compile tests/cpp/<name>.cpp against libtrajopt_b200, once per session: an executable, or with `shared` a shared
    library.  `extra`: more compiler and linker arguments, after the common ones."""
    key = (name, shared, tuple(extra))
    if key not in _built:
        capi.load_library()  # the CUDA build must exist (no GPU needed to load it)
        out = str(tmp_path_factory.mktemp(name) / (f"lib{name}.so" if shared else name))
        cmd = ["g++", "-std=c++17", "-O1", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"),
               os.path.join(ROOT, "tests", "cpp", name + ".cpp"), "-o", out, "-L", CSRC, "-ltrajopt_b200",
               "-Wl,-rpath," + CSRC, "-Wl,--allow-shlib-undefined", *(["-shared", "-fPIC"] if shared else []), *extra]
        subprocess.run(cmd, check=True)
        _built[key] = out
    return _built[key]


def write_problem(path, desc):
    """Write desc's robot, trajectories, first cart target of every trajectory (the one of configs[2]; none when desc has
    none) and obstacles as the host programs read them; the links are named link<segment index>.  Returns the path as a
    string."""
    robot = desc.robot_spec
    names = [f"link{i}" for i in range(len(robot["segments"]))]
    targets = np.zeros((0, 7)) if desc.cart_targets is None else desc.cart_targets[:, 0]
    num = lambda vals: " ".join(repr(float(v)) for v in vals)  # noqa: E731  (repr: the shortest exact decimal)
    with open(path, "w") as f:
        f.write(f"{desc.B} {desc.T} {desc.D} {len(names)}\n")
        for name, s in zip(names, robot["segments"]):
            f.write(f"{s.parent} {s.joint_type} {s.q_index} {num([*s.origin_xyz, *s.origin_wxyz, *s.axis])} {name}\n")
        f.write(num(robot["lower"]) + "\n" + num(robot["upper"]) + "\n")
        f.write(f"{len(robot['spheres'])}\n")
        for sp in robot["spheres"]:
            f.write(f"{names[sp.segment]} {num([*sp.center, sp.radius])}\n")
        f.write(names[robot["tool"]] + "\n")
        f.write(num(desc.init_traj.ravel()) + "\n")
        f.write(f"{len(targets)}\n{num(targets.ravel())}\n")
        f.write(f"{desc.obstacles.shape[1]}\n{num(desc.obstacles.ravel())}\n")
    return str(path)
