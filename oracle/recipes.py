"""TEST INFRASTRUCTURE — how every library under oracle/ is compiled: one table with one row per library, and the small
engine that runs it.  Nothing else under oracle/ runs a compiler.

    python -m oracle.recipes [--ref DIR] [--force] [--dry-run]

builds every plain-C restatement library that is out of date and, with --ref naming a checkout of the original project,
every reference library whose files that checkout has: the unmodified sources compiled where they lie, against the
stand-ins under oracle/shim*/.  Outputs go to oracle/ and oracle/_ref/ (git-ignored); nothing is copied out of the
checkout.  --force rebuilds what is up to date; --dry-run prints the commands instead of running them.

Paths in the table are relative to oracle/, or to the reference checkout where they start with $REF.  An include
directory is written where its -I flag goes on the command line.
"""
from __future__ import annotations

import argparse
import os
import re
import shlex
import subprocess
from dataclasses import dataclass

ORACLE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(ORACLE)
REF = "$REF"

# Every row builds for the x86-64 baseline, with no -march, so no FMA contraction: like the reference's catkin build.
C_FLAGS = ["-O2", "-fPIC", "-std=c11", "-ffp-contract=off", "-Wall", "-Wextra"]  # the restatements
REF_C_FLAGS = ["-std=c11", "-O2", "-fPIC", "-w", "-ffp-contract=off"]  # a restatement linked into a reference library
CXX_FLAGS = ["-std=c++17", "-O2", "-fPIC", "-w"]  # the reference
REF_CXX_FLAGS = CXX_FLAGS + ["-ffp-contract=off"]


@dataclass(frozen=True)
class Step:
    """One compiler call: flags, then sources.  A compile-only step makes an object (-c) that the row's last step links
    after its own sources."""
    lang: str  # "c" or "c++"
    flags: tuple
    sources: tuple = ()
    compile_only: bool = False


@dataclass(frozen=True)
class Recipe:
    out: str
    steps: tuple
    link: tuple = ()  # after -o <out> on the last step
    # False: plain gcc / g++ from PATH, not $CC / $CXX.  A reference library that runs C++ is loaded next to numpy's
    # libstdc++, and a newer compiler's inline libstdc++ code does not mix with it.
    env_compiler: bool = True
    ref_files: tuple = ()  # the checkout's files the sources #include; with the $REF sources, they gate the build


def _one(out, lang, flags, sources, link=("-lm",), **kw) -> Recipe:
    """A library made by one compiler call."""
    return Recipe(out, (Step(lang, tuple(flags), tuple(sources)),), tuple(link), **kw)


_L4 = "-I$REF/lesson4/include"
_KARTO = ("$REF/lesson6/lib/open_karto/src/Karto.cpp", "$REF/lesson6/lib/open_karto/src/Mapper.cpp")

TABLE = (
    # ---- the plain-C restatements, always built
    _one("libslam_oracle.so", "c", C_FLAGS + ["-shared"],
         ["karto_oracle.c", "gmapping_oracle.c", "hector_oracle.c", "plicp_oracle.c", "deskew_oracle.c"],
         env_compiler=False),  # plain gcc
    _one("libpcl_icp_oracle.so", "c", C_FLAGS + ["-shared"], ["pcl_icp_oracle.c"]),
    _one("libfeature_oracle.so", "c++",
         ["-std=c++17", "-O2", "-fPIC", "-ffp-contract=off", "-Wall", "-Wextra", "-shared"], ["feature_oracle.cpp"],
         link=()),
    _one("libplicp_odometry_oracle.so", "c", C_FLAGS + ["-shared"], ["plicp_odometry_oracle.c", "plicp_oracle.c"]),
    _one("libplicp_scan_match_oracle.so", "c", C_FLAGS + ["-shared"], ["plicp_scan_match_oracle.c", "plicp_oracle.c"]),
    _one("liblesson4_nodes_oracle.so", "c", C_FLAGS + ["-shared"],
         ["lesson4_nodes_oracle.c", "gmapping_oracle.c", "hector_oracle.c"]),
    _one("libdeskew_node_oracle.so", "c", C_FLAGS + ["-D_DEFAULT_SOURCE", "-shared"],
         ["deskew_node_oracle.c", "deskew_oracle.c"]),  # -D_DEFAULT_SOURCE: this row only
    # ---- the unmodified reference, built where a checkout of it is given
    _one("_ref/libkarto_ref.so", "c++", CXX_FLAGS + ["-shared", "-Ishim", "-I$REF/lesson6/lib/open_karto/include"],
         ["ref_driver.cpp", *_KARTO], link=(), env_compiler=False),  # no -ffp-contract=off; plain g++
    _one("_ref/libkarto_ref_ndebug.so", "c++",  # the timing build: the flags BASELINE.md names (-O2 -DNDEBUG)
         CXX_FLAGS + ["-DNDEBUG", "-shared", "-Ishim", "-I$REF/lesson6/lib/open_karto/include"],
         ["ref_driver.cpp", *_KARTO], link=(), env_compiler=False),  # -DNDEBUG; no -ffp-contract=off; plain g++
    _one("_ref/libgmapping_ref.so", "c++", CXX_FLAGS + ["-DNDEBUG", "-shared", _L4], ["ref_gmapping.cpp"], link=(),
         env_compiler=False,  # -DNDEBUG; no -ffp-contract=off; plain g++
         ref_files=("$REF/lesson4/include/lesson4/gmapping/grid/map.h",
                    "$REF/lesson4/include/lesson4/gmapping/grid/gridlinetraversal.h")),
    _one("_ref/libhector_ref.so", "c++", REF_CXX_FLAGS + ["-shared", "-Ishim", _L4], ["ref_hector.cpp"], link=(),
         env_compiler=False,  # plain g++
         ref_files=("$REF/lesson4/include/lesson4/hector_mapping/slam_main/HectorSlamProcessor.h",)),
    _one("_ref/liblesson1_ref.so", "c++", CXX_FLAGS + ["-shared", "-Ishim", "-I$REF"], ["ref_lesson1.cpp"], link=(),
         ref_files=("$REF/lesson1/src/feature_detection.cc",)),  # no -ffp-contract=off
    _one("_ref/liblesson5_ref.so", "c++", REF_CXX_FLAGS + ["-shared", "-Ishim", "-I$REF", "-I$REF/lesson5/include"],
         ["ref_lesson5.cpp"], link=(),
         ref_files=("$REF/lesson5/src/lidar_undistortion.cc", "$REF/lesson5/include/lesson5/lidar_undistortion.h")),
    Recipe("_ref/liblesson3_ref.so",
           (Step("c", tuple(REF_C_FLAGS), ("plicp_oracle.c",), compile_only=True),
            Step("c++", tuple(REF_CXX_FLAGS + ["-shared", "-Ishim", "-I$REF", "-I$REF/lesson3/include"]),
                 ("ref_lesson3.cpp",))), ("-lm",),
           ref_files=("$REF/lesson3/src/plicp_odometry.cc", "$REF/lesson3/include/lesson3/plicp_odometry.h")),
    Recipe("_ref/liblesson3_scan_match_ref.so",
           (Step("c", tuple(REF_C_FLAGS), ("plicp_oracle.c",), compile_only=True),
            Step("c++", tuple(REF_CXX_FLAGS + ["-shared", "-Ishim", "-I$REF", "-I$REF/lesson3/include"]),
                 ("ref_lesson3_scan_match.cpp",))), ("-lm",),
           ref_files=("$REF/lesson3/src/scan_match_plicp.cc", "$REF/lesson3/include/lesson3/scan_match_plicp.h")),
    Recipe("_ref/liblesson4_ref.so",  # two translation units: see ref_lesson4_hector.cpp
           tuple(Step("c++", tuple(REF_CXX_FLAGS + ["-Ishim", "-I$REF", _L4, _L4 + "/lesson4/hector_mapping"]), (d,),
                      compile_only=True) for d in ("ref_lesson4_gmapping.cpp", "ref_lesson4_hector.cpp")) +
           (Step("c++", ("-shared",)),), ("-lm",),
           ref_files=("$REF/lesson4/src/gmapping/gmapping.cc", "$REF/lesson4/src/hector_mapping/hector_mapping.cc")),
    _one("_ref/liblesson4_slam_ref.so", "c++",
         REF_CXX_FLAGS + ["-Ishim_lesson4_slam", "-Ishim_lesson6", "-Ishim", "-I$REF", _L4,
                          _L4 + "/lesson4/hector_mapping", "-shared"],
         ["ref_lesson4_slam.cpp"], ref_files=("$REF/lesson4/src/hector_mapping/hector_slam.cc",)),
    _one("_ref/liblesson6_ref.so", "c++",
         REF_CXX_FLAGS + ["-shared", "-Ishim_lesson6", "-Ishim", "-I$REF", "-I$REF/lesson6/include",
                          "-I$REF/lesson6/lib/open_karto/include"],
         ["ref_lesson6.cpp", *_KARTO], env_compiler=False,  # plain g++
         ref_files=("$REF/lesson6/src/karto_slam.cc", "$REF/lesson6/include/lesson6/karto_slam.h")),
)
RECIPES = {r.out: r for r in TABLE}


def path(name: str) -> str:
    return os.path.join(ORACLE, name)


def available(name: str) -> bool:
    return os.path.exists(path(name))


def _resolve(p: str, ref) -> str:
    if not p.startswith(REF):
        return os.path.join(ORACLE, p)
    if ref is None:
        raise ValueError(f"{p} is in the reference checkout, and none was given")
    return os.path.abspath(ref) + p[len(REF):]


def _flag(f: str, ref) -> str:
    return "-I" + _resolve(f[2:], ref) if f.startswith("-I") else f


def _reference_files(r: Recipe) -> list:
    return [p for s in r.steps for p in s.sources if p.startswith(REF)] + list(r.ref_files)


_INCLUDE = re.compile(r'^[ \t]*#[ \t]*include[ \t]*([<"])([^>"]+)[>"]', re.M)


def deps(name: str, ref=None) -> list:
    """Every file the library is made from: its sources, every file under its oracle-side include directories, every
    file its sources reach through #include (through the reference checkout's files too, when `ref` is given), its
    reference files and this module."""
    r = RECIPES[name]
    inc = [f[2:] for s in r.steps for f in s.flags if f.startswith("-I")]
    out = {os.path.join(top, f) for d in inc if not d.startswith(REF) for top, _, files in os.walk(_resolve(d, ref))
           for f in files}
    dirs = [_resolve(d, ref) for d in inc if ref is not None or not d.startswith(REF)]
    todo = [_resolve(p, ref) for s in r.steps for p in s.sources if ref is not None or not p.startswith(REF)]
    seen = set()
    while todo:
        f = os.path.normpath(todo.pop())
        if f in seen:
            continue
        seen.add(f)
        with open(f, errors="replace") as fh:
            for kind, inc in _INCLUDE.findall(fh.read()):
                for d in ([os.path.dirname(f)] if kind == '"' else []) + dirs:
                    if os.path.isfile(os.path.join(d, inc)):
                        todo.append(os.path.join(d, inc))
                        break
    if ref is not None:
        out.update(_resolve(p, ref) for p in r.ref_files)
    return sorted(out | seen | {os.path.abspath(__file__)})


def stale(name: str, ref=None) -> bool:
    out = path(name)
    if not os.path.exists(out):
        return True
    t = os.path.getmtime(out)
    return any(os.path.getmtime(d) > t for d in deps(name, ref))


def commands(name: str, ref=None, tmp=None):
    """-> (the compiler calls that make the library at `tmp`, the objects they leave beside it)."""
    r = RECIPES[name]
    tmp = tmp or path(name) + f".{os.getpid()}.tmp"
    cmds, objs = [], []
    for s in r.steps:
        cc = (os.environ.get("CC", "gcc") if r.env_compiler else "gcc") if s.lang == "c" else \
            (os.environ.get("CXX", "g++") if r.env_compiler else "g++")
        argv = [cc] + [_flag(f, ref) for f in s.flags]
        srcs = [_resolve(p, ref) for p in s.sources]
        if s.compile_only:
            objs.append(f"{tmp}.{os.path.basename(s.sources[0])}.o")
            cmds.append(argv + ["-c"] + srcs + ["-o", objs[-1]])
        else:
            cmds.append(argv + srcs + objs + ["-o", tmp] + list(r.link))
    return cmds, objs


def build(name: str, ref=None, force: bool = False, dry_run: bool = False) -> str:
    """Make the library `name` unless it is up to date; `ref` is the reference checkout a reference library needs.
    The compiler writes <out>.<pid>.tmp, which replaces <out> at once: a concurrent reader sees the old library or the
    new one."""
    out = path(name)
    if not force and not stale(name, ref):
        return out
    tmp = out + f".{os.getpid()}.tmp"
    cmds, objs = commands(name, ref, tmp)
    if dry_run:
        for c in cmds:
            print(shlex.join(c))
        return out
    os.makedirs(os.path.dirname(out), exist_ok=True)
    try:
        for c in cmds:
            subprocess.check_call(c)
        os.replace(tmp, out)
    finally:
        for f in objs + [tmp]:
            if os.path.exists(f):
                os.remove(f)
    return out


def build_all(ref=None, force: bool = False, dry_run: bool = False) -> None:
    """Every restatement library, and with `ref` every reference library whose reference files the checkout has."""
    for name, r in RECIPES.items():
        files = _reference_files(r)
        if not files or (ref is not None and all(os.path.isfile(_resolve(p, ref)) for p in files)):
            build(name, ref, force, dry_run)


def main(argv=None) -> None:
    ap = argparse.ArgumentParser(prog="python -m oracle.recipes", description="Build the oracle libraries.")
    ap.add_argument("--ref", help="a checkout of the original project: build the reference libraries too")
    ap.add_argument("--force", action="store_true", help="rebuild libraries that are up to date")
    ap.add_argument("--dry-run", action="store_true", help="print the commands that would run, and run none")
    a = ap.parse_args(argv)
    build_all(a.ref, a.force, a.dry_run)


if __name__ == "__main__":
    main()
