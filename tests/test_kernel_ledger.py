"""The kernel ledger (tests/_kernel_ledger.py) against the built library: the instances ``nm -C`` (or ``cuobjdump -res-usage``)
lists are exactly the ledger's, and every instance the ledger gives to tests/test_kernel_ledger_gpu.py names one of that
file's test functions.  No GPU needed."""
import ast
import os
import re
import shutil
import subprocess

import pytest

from tests import _kernel_ledger as K

ROOT = K.ROOT
LIB = os.path.join(ROOT, "torchx_b200", "lib", "libb200ddp.so")


def normalise(demangled):
    """A demangled kernel symbol as tools/sass_report.demangle prints it: no anonymous namespace, return type or parameters."""
    d = re.sub(r"\(anonymous namespace\)::", "", demangled.strip())
    d = re.sub(r"^void ", "", d)
    return re.sub(r"\(.*$", "", d)


def library_kernels():
    """The kernel instances of the built library, or skip."""
    if not os.path.isfile(LIB):
        pytest.skip("libb200ddp.so is not built")
    if shutil.which("nm"):
        out = subprocess.run(["nm", "-C", LIB], capture_output=True, text=True, check=True).stdout
        # "<address> <type> <demangled symbol>": the host stub of each __global__ function carries the kernel's name
        names = {normalise(line.split(" ", 2)[2]) for line in out.splitlines() if len(line.split(" ", 2)) == 3}
    elif shutil.which("cuobjdump") and shutil.which("c++filt"):
        out = subprocess.run(["cuobjdump", "-res-usage", LIB], capture_output=True, text=True, check=True).stdout
        mangled = re.findall(r"^\s*Function (\S+):", out, flags=re.M)
        dem = subprocess.run(["c++filt"], input="\n".join(mangled), capture_output=True, text=True, check=True).stdout
        names = {normalise(d) for d in dem.splitlines()}
    else:
        pytest.skip("neither nm nor cuobjdump is available")
    return {n for n in names if re.fullmatch(r"k_\w+(<[^>]*>)?", n)}


def test_ledger_is_built_from_the_header():
    assert K.MAX_WORLD == 8 and list(K.WORLDS) == list(range(2, 9))
    assert K.MODES == [0, 1, 2, 3, 4]
    assert len(K.EXACT) == 12


def test_library_holds_exactly_the_ledgers_kernels():
    got = library_kernels()
    want = set(K.LEDGER)
    missing, extra = sorted(want - got), sorted(got - want)
    assert not missing, f"{len(missing)} ledger instances are not in the library: {missing}"
    assert not extra, f"{len(extra)} kernel instances of the library have no ledger entry (and no test that launches them): {extra}"
    assert len(got) == 321, len(got)
    print(f"{len(got)} kernel instances, the ledger equals the library's list")


def _test_functions(path):
    tree = ast.parse(open(os.path.join(ROOT, path)).read())
    return [n.name for n in tree.body if isinstance(n, ast.FunctionDef) and n.name.startswith("test_")]


def test_every_entry_names_a_test_that_exists():
    funcs = _test_functions(K.NEW)
    for name, where in K.LEDGER.items():
        if where == K.MULTICAST:
            continue
        path, _, fn = where.partition("::")
        assert os.path.isfile(os.path.join(ROOT, path)), (name, where)
        if path == K.NEW:
            assert funcs.count(fn) == 1, f"{name}: {where} is not exactly one test function of {K.NEW}"
        else:
            assert not fn, (name, where)
            assert _test_functions(path), (name, where)


def test_the_new_gpu_file_owns_the_instances_no_older_test_launches():
    """60 instances at W = 5, 6, 7 that one device can run, and the six BatchNorm2d kernels at C > 2048."""
    mine = {n for n, w in K.LEDGER.items() if w.startswith(K.NEW + "::")}
    bn = {n for n in mine if n.startswith("k_bn2d_")}
    assert len(bn) == 6
    rest = mine - bn
    assert len(rest) == 60, len(rest)
    assert {K.template_args(n)[1] for n in rest} == set(K.NEW_WORLDS)
    nvls = {n for n, w in K.LEDGER.items() if w == K.MULTICAST}
    assert nvls == {f"k_pipe<{m}, {W}, {K.K_NVLS}>" for m in K.MODES for W in K.WORLDS}
