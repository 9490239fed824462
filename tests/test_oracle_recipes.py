"""The oracle libraries' recipe table (oracle/recipes.py): every row names files that exist, its derived dependencies
cover every header the compiler reads, it runs the command it is meant to, and no other oracle module runs a compiler.
CPU only; no reference checkout needed (reference rows are preprocessed against an empty stand-in for it); nothing in
the repository is written."""
import glob
import os
import re
import shlex
import subprocess

import pytest

from oracle import recipes

O = recipes.ORACLE


def _in_repo(p):
    return os.path.realpath(p).startswith(recipes.ROOT + os.sep)


def test_rows_name_existing_files_and_unique_outputs():
    assert len({r.out for r in recipes.TABLE}) == len(recipes.TABLE) == len(recipes.RECIPES)
    for r in recipes.TABLE:
        assert r.steps and not r.steps[-1].compile_only, r.out
        for s in r.steps:
            assert s.lang in ("c", "c++"), r.out
            for p in s.sources:
                assert p.startswith(recipes.REF) or os.path.isfile(os.path.join(O, p)), (r.out, p)
            for f in s.flags:
                if f.startswith("-I") and not f[2:].startswith(recipes.REF):
                    assert os.path.isdir(os.path.join(O, f[2:])), (r.out, f)
        assert all(p.startswith(recipes.REF + "/") for p in r.ref_files), r.out


@pytest.mark.parametrize("name", list(recipes.RECIPES))
def test_deps_cover_every_header_the_compiler_reads(name, tmp_path):
    """`cc -M -MG` on each compile step of the row: every file it reads inside the repository is a dependency."""
    cmds, _ = recipes.commands(name, str(tmp_path), tmp=str(tmp_path / "out"))
    dep = {os.path.realpath(d) for d in recipes.deps(name)}
    read = set()
    for c in cmds:
        srcs = [t for t in c[1:] if t.endswith((".c", ".cpp")) and _in_repo(t)]
        flags = [t for t in c[1:] if t.startswith("-") and t not in ("-shared", "-c", "-o") and not t.startswith("-l")]
        if srcs:
            out = subprocess.run([c[0], *flags, "-M", "-MG", *srcs], capture_output=True, text=True, check=True).stdout
            words = out.replace("\\\n", " ").split()
            read |= {os.path.realpath(os.path.join(O, t)) for t in words if not t.endswith(":")}
    read = {f for f in read if _in_repo(f) and os.path.isfile(f)}
    assert read and read <= dep, sorted(read - dep)
    assert os.path.realpath(recipes.__file__) in dep
    if name == "libslam_oracle.so":
        assert os.path.join(recipes.ROOT, "include", "b200slam.h") in dep


def test_only_recipes_runs_a_compiler():
    for f in glob.glob(os.path.join(O, "*.py")):
        if os.path.basename(f) == "recipes.py":
            continue
        src = open(f).read()
        assert "subprocess" not in src, f
        assert not re.search(r'\b(gcc|g\+\+|clang\+*|nvcc)\b|"CC"|"CXX"', src), f


def test_dry_run_prints_each_rows_command(tmp_path, capsys):
    ref = tmp_path / "reference"
    for p in recipes.RECIPES["_ref/liblesson3_ref.so"].ref_files:
        (ref / p[len("$REF/"):]).parent.mkdir(parents=True, exist_ok=True)
        (ref / p[len("$REF/"):]).write_text("")
    recipes.main(["--ref", str(ref), "--force", "--dry-run"])
    lines = capsys.readouterr().out.splitlines()
    pid, R = os.getpid(), str(ref)
    slam = f"{O}/libslam_oracle.so.{pid}.tmp"
    l3 = f"{O}/_ref/liblesson3_ref.so.{pid}.tmp"
    cc, cxx = os.environ.get("CC", "gcc"), os.environ.get("CXX", "g++")
    want = [
        ["gcc", "-O2", "-fPIC", "-std=c11", "-ffp-contract=off", "-Wall", "-Wextra", "-shared",
         *(f"{O}/{s}" for s in ("karto_oracle.c", "gmapping_oracle.c", "hector_oracle.c", "plicp_oracle.c",
                                "deskew_oracle.c")), "-o", slam, "-lm"],
        [cc, "-std=c11", "-O2", "-fPIC", "-w", "-ffp-contract=off", "-c", f"{O}/plicp_oracle.c",
         "-o", f"{l3}.plicp_oracle.c.o"],
        [cxx, "-std=c++17", "-O2", "-fPIC", "-w", "-ffp-contract=off", "-shared", f"-I{O}/shim", f"-I{R}",
         f"-I{R}/lesson3/include", f"{O}/ref_lesson3.cpp", f"{l3}.plicp_oracle.c.o", "-o", l3, "-lm"],
    ]
    for w in want:
        assert shlex.join(w) in lines
    # every restatement, and of the reference libraries only the one whose files the checkout has
    built = {re.search(r" -o (\S+)\.\d+\.tmp( |$)", ln).group(1) for ln in lines if re.search(r"\.\d+\.tmp( |$)", ln)}
    restatements = {recipes.path(r.out) for r in recipes.TABLE if not r.out.startswith("_ref/")}
    assert built == restatements | {recipes.path("_ref/liblesson3_ref.so")}
    assert not glob.glob(os.path.join(O, "**", f"*.{pid}.tmp*"), recursive=True)
