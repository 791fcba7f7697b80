"""Compiles the C++ test programs under tests/cpp, all with one command line."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB_DIRS = {"famsa_b200": os.path.join(ROOT, "famsa_b200", "lib"), "oracle": os.path.join(ROOT, "oracle")}


def build_cpp(name: str, out_dir, famsa: bool = False, oracle: bool = False) -> str:
    """tests/cpp/<name>.cpp built into out_dir/<name>, linked against libfamsa_b200.so and / or oracle/liboracle.so
    (each found at run time through an rpath).  Returns the executable's path."""
    exe = os.path.join(str(out_dir), name)
    cmd = ["g++", "-std=c++17", "-O1", "-Wall", "-Werror", os.path.join(ROOT, "tests", "cpp", name + ".cpp"), "-o", exe]
    for lib, wanted in (("famsa_b200", famsa), ("oracle", oracle)):
        if wanted:
            cmd += ["-L" + LIB_DIRS[lib], "-l" + lib, "-Wl,-rpath," + LIB_DIRS[lib]]
    subprocess.run(cmd, check=True)
    return exe
