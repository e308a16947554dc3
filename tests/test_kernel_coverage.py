"""Every C entry point of the library is exercised by a GPU test, directly or through a Python wrapper.

The entry points are the `int mg_*(` / `long long mg_*(` declarations of include/michigan_b200.h.  A tests/test_gpu_*.py module
exercises one when its code (not its comments or docstrings) names the entry point itself, an ops.* wrapper that calls it
(directly or through other ops.* functions), or a top-level class / function of the package that reaches it (e.g.
SpectralNormBatch, LabColorLoss; not a whole network, see END_TO_END).  Package names count only as the module's imports
bind them.  Entry points no such module reaches are listed in NOT_IN_GPU_TESTS with the reason.

Every hand-written backward function of the training path is reached by tests/test_gpu_backward_stages_fp64.py, which holds
each stage to float64 autograd element by element; functions deliberately left out are listed in NOT_IN_BACKWARD_STAGES.
"""
import ast
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "michigan_b200.h")
PKG = os.path.join(ROOT, "michigan_b200")
TESTS = os.path.join(ROOT, "tests")

ENTRY_RE = re.compile(r"^\s*(?:int|long\s+long)\s+(mg_\w+)\s*\(", re.M)

NOT_IN_GPU_TESTS = {
    "mg_peer_allreduce_f64": "needs two GPUs: tests/nccl_worker.py runs it on 2 GPUs (launched by test_gpu_multi.py)",
    "mg_peer_buffer_bytes": "size query of the 2-GPU all-reduce, called by tests/nccl_worker.py on 2 GPUs",
    "mg_peer_max_elems": "size query of the 2-GPU all-reduce, called by tests/nccl_worker.py on 2 GPUs",
    "mg_debug_seg_prof": "probe counters, compiled only into the -DMG_PROBES build that tools/ load",
    "mg_version": "ABI query, checked by tests/test_abi.py",
    "mg_launch_count": "ABI query, checked by tests/test_abi.py",
    "mg_set_tuning": "ABI knob setter, checked by tests/test_abi.py",
    "mg_get_tuning": "ABI knob getter, checked by tests/test_abi.py",
    "mg_style_tap_bytes": "descriptor size query, checked against the ctypes layout by tests/test_abi.py",
}


# Tests that hold a kernel's every output element to a float64 reference (under a per-element bound) or to the bits of an
# exact restatement.  Whole modules of such tests, then the named tests of modules that also hold end-to-end checks.
ELEMENTWISE_MODULES = [
    "test_gpu_backward_kernels.py",
    "test_gpu_conv_forward_fp64.py",
    "test_gpu_cuda_core_forward_fp64.py",
    "test_gpu_loss_kernels_fp64.py",
]
ELEMENTWISE_TESTS = {
    "test_gpu_style_content.py": ["test_style_kernels_vs_fp64_autograd", "test_pixel_l1_vs_fp64_autograd",
                                  "test_content_op3_vs_fp64_autograd"],
    "test_gpu_hair_avg_lab.py": ["test_hair_avg_lab_kernels_vs_fp64_autograd"],
    "test_gpu_vgg_lab.py": ["test_maxpool2_forward_backward_vs_torch"],
}
# Entry points outside NOT_IN_GPU_TESTS that no element-wise test reaches, with the reason (none today).
NOT_ELEMENTWISE = {}


# The module that holds every hand-written backward stage to float64 autograd, and the backward functions it leaves out.
BACKWARD_STAGES_MODULE = "test_gpu_backward_stages_fp64.py"
NOT_IN_BACKWARD_STAGES = {
    "_GeneratorFn.backward": "chains conv_img_bwd (test_gpu_backward_kernels.py) and the stages block_bwd, latent_bwd, "
                             "backward_nhwc and bg_bwd, each tested on its own; end to end in test_gpu_parity.py",
    "_ConvEncoderFn.backward": "concatenates d mu | d logvar and calls conv_encoder_bwd, which is tested; end to end in "
                               "test_gpu_vae.py",
}


# Whole networks and the training model run dozens of kernels end to end, under bounds loose enough to pass a kernel that is
# wrong on one border or channel range: reaching an entry point only through one of them does not count.
END_TO_END = {"BaseNetwork", "Pix2PixModel"}
# Code that runs only across two or more ranks (single-process callers return before reaching it): reaching it credits nothing.
MULTI_RANK = {"_PeerExchange"}


def entry_points():
    with open(HEADER) as f:
        return set(ENTRY_RE.findall(f.read()))


def _code_names(tree):
    """Identifiers a module's code uses: names and attribute names (strings, comments and docstrings do not count)."""
    out = set()
    for node in ast.walk(tree):
        if isinstance(node, ast.Name):
            out.add(node.id)
        elif isinstance(node, ast.Attribute):
            out.add(node.attr)
        elif isinstance(node, ast.alias):
            out.add(node.name.split(".")[-1])
    return out


def _parse(path):
    with open(path) as f:
        src = f.read()
    return src, ast.parse(src)


def ops_wrappers():
    """ops.<function> -> entry points it calls, following calls to other ops functions."""
    src, tree = _parse(os.path.join(PKG, "ops.py"))
    funcs = {n.name: n for n in tree.body if isinstance(n, ast.FunctionDef)}
    direct = {name: {a for a in _code_names(fn) if a.startswith("mg_")} for name, fn in funcs.items()}
    calls = {name: {n.func.id for n in ast.walk(fn) if isinstance(n, ast.Call) and isinstance(n.func, ast.Name)
                    and n.func.id in funcs} for name, fn in funcs.items()}
    out = {}
    for name in funcs:
        seen, todo, eps = set(), [name], set()
        while todo:
            f = todo.pop()
            if f in seen:
                continue
            seen.add(f)
            eps |= direct[f]
            todo.extend(calls[f])
        out[name] = eps
    return out


def package_callers():
    """Top-level classes and functions of the other package modules -> entry points their code reaches: the ones it names,
    those of the ops.* wrappers it calls, and those of the other top-level classes / functions it uses."""
    wrappers = ops_wrappers()
    uses = {}
    for dirpath, _, files in os.walk(PKG):
        for fn in files:
            if not fn.endswith(".py") or fn in ("ops.py", "_lib.py"):
                continue
            _, tree = _parse(os.path.join(dirpath, fn))
            for node in tree.body:
                if isinstance(node, ast.ClassDef) and (node.name in END_TO_END | MULTI_RANK or
                                                       any(getattr(bs, "id", None) in END_TO_END for bs in node.bases)):
                    continue
                if isinstance(node, (ast.ClassDef, ast.FunctionDef)):
                    uses.setdefault(node.name, set()).update(_code_names(node))
    out = {}
    for name in uses:
        seen, todo, eps = set(), [name], set()
        while todo:
            n = todo.pop()
            if n in seen:
                continue
            seen.add(n)
            for m in uses[n]:
                if m.startswith("mg_"):
                    eps.add(m)
                elif m in uses:
                    todo.append(m)
                else:
                    eps |= wrappers.get(m, set())
        out[name] = eps
    return out


def _is_package_module(dotted):
    rel = os.path.join(ROOT, *dotted.split("."))
    return os.path.isfile(rel + ".py") or os.path.isfile(os.path.join(rel, "__init__.py"))


def _local_scope(tree, names):
    """The module-level functions `names` and every module-level function or class they call by name, transitively."""
    defs = {n.name: n for n in tree.body if isinstance(n, (ast.FunctionDef, ast.ClassDef))}
    seen, todo = set(), [n for n in names if n in defs]
    while todo:
        n = todo.pop()
        if n in seen:
            continue
        seen.add(n)
        todo.extend(m for m in _code_names(defs[n]) if m in defs)
    return [defs[n] for n in sorted(seen)]


def _test_module_reach(tree, wrappers, callers, scope=None):
    """Entry points a test module's code reaches, resolving names through its imports only: `mg_*` attributes (calls into
    the loaded library), package modules bound by an import (also through a local getter such as `def _ops(): from
    michigan_b200 import ops; return ops` and `ops = _ops()`) and their attributes, and classes / functions imported from
    the package.  A local variable that happens to share a package name is not a package reference.  With `scope` (a list
    of nodes of the module), only the code of those nodes counts; the imports are still resolved over the whole module."""
    modules, symbols = {}, {}
    for node in ast.walk(tree):
        if isinstance(node, ast.ImportFrom) and node.module and node.module.split(".")[0] == "michigan_b200":
            for a in node.names:
                full = node.module + "." + a.name
                if _is_package_module(full):
                    modules[a.asname or a.name] = full
                else:
                    symbols[a.asname or a.name] = (node.module, a.name)
        elif isinstance(node, ast.Import):
            for a in node.names:
                if a.name.split(".")[0] == "michigan_b200" and a.asname:
                    modules[a.asname] = a.name
    getters = {}
    for node in ast.walk(tree):
        if isinstance(node, ast.FunctionDef):
            for r in ast.walk(node):
                if isinstance(r, ast.Return) and isinstance(r.value, ast.Name) and r.value.id in modules:
                    getters[node.name] = modules[r.value.id]

    def module_of(expr):
        if isinstance(expr, ast.Name):
            return modules.get(expr.id)
        if isinstance(expr, ast.Call) and isinstance(expr.func, ast.Name):
            return getters.get(expr.func.id)
        return None

    for node in ast.walk(tree):
        if isinstance(node, ast.Assign):
            pairs = [(node.targets[0], node.value)]
            if isinstance(node.targets[0], ast.Tuple) and isinstance(node.value, ast.Tuple):
                pairs = list(zip(node.targets[0].elts, node.value.elts))
            for t, v in pairs:
                m = module_of(v)
                if m and isinstance(t, ast.Name):
                    modules[t.id] = m

    def resolve(module, name):
        return wrappers.get(name, set()) if module == "michigan_b200.ops" else callers.get(name, set())

    eps = set()
    for node in (n for s in (scope if scope is not None else [tree]) for n in ast.walk(s)):
        if isinstance(node, ast.Attribute):
            if node.attr.startswith("mg_"):
                eps.add(node.attr)
            m = module_of(node.value)
            if m:
                eps |= resolve(m, node.attr)
        elif isinstance(node, ast.Name) and node.id in symbols:
            eps |= resolve(*symbols[node.id])
    return eps


def exercised_by_gpu_tests():
    """entry point -> the tests/test_gpu_*.py modules whose code reaches it."""
    wrappers, callers = ops_wrappers(), package_callers()
    reach = {}
    for fn in sorted(os.listdir(TESTS)):
        if not (fn.startswith("test_gpu_") and fn.endswith(".py")):
            continue
        _, tree = _parse(os.path.join(TESTS, fn))
        for e in _test_module_reach(tree, wrappers, callers):
            reach.setdefault(e, set()).add(fn)
    return reach


def test_header_lists_the_entry_points():
    eps = entry_points()
    assert len(eps) > 50, sorted(eps)
    assert {"mg_conv_igemm", "mg_bn_stats", "mg_spectral_norm_batched", "mg_peer_allreduce_f64"} <= eps


def test_ops_wrappers_call_declared_entry_points():
    eps = entry_points()
    w = ops_wrappers()
    assert w["mlp_shared"] >= {"mg_conv_seg_tc", "mg_conv_thin"}
    undeclared = {n: sorted(e - eps) for n, e in w.items() if e - eps}
    assert not undeclared, undeclared


def test_every_header_entry_point_is_exercised_by_a_gpu_test():
    eps = entry_points()
    reach = exercised_by_gpu_tests()
    assert set(NOT_IN_GPU_TESTS) <= eps, sorted(set(NOT_IN_GPU_TESTS) - eps)
    missing = sorted(e for e in eps if e not in reach and e not in NOT_IN_GPU_TESTS)
    assert not missing, "entry points no tests/test_gpu_*.py module reaches (add a test or list them with a reason): %s" % missing
    stale = sorted(e for e in NOT_IN_GPU_TESTS if e in reach)
    assert not stale, "listed as untested but reached by a GPU test: %s" % stale


def exercised_by_elementwise_tests():
    """entry point -> the element-wise tests (module, or module::function) whose code reaches it."""
    wrappers, callers = ops_wrappers(), package_callers()
    reach = {}
    for fn in sorted(set(ELEMENTWISE_MODULES) | set(ELEMENTWISE_TESTS)):
        _, tree = _parse(os.path.join(TESTS, fn))
        if fn in ELEMENTWISE_MODULES:
            scopes = {fn: None}
        else:
            defs = {n.name for n in tree.body if isinstance(n, ast.FunctionDef)}
            missing = sorted(set(ELEMENTWISE_TESTS[fn]) - defs)
            assert not missing, "%s has no test %s" % (fn, missing)
            scopes = {fn + "::" + t: _local_scope(tree, [t]) for t in ELEMENTWISE_TESTS[fn]}
        for name, scope in scopes.items():
            for e in _test_module_reach(tree, wrappers, callers, scope):
                reach.setdefault(e, set()).add(name)
    return reach


def test_every_entry_point_has_an_elementwise_test():
    eps = entry_points()
    reach = exercised_by_elementwise_tests()
    for fn in set(ELEMENTWISE_MODULES) | set(ELEMENTWISE_TESTS):
        assert os.path.isfile(os.path.join(TESTS, fn)), "element-wise test module %s is missing" % fn
    assert set(NOT_ELEMENTWISE) <= eps, sorted(set(NOT_ELEMENTWISE) - eps)
    missing = sorted(e for e in eps if e not in reach and e not in NOT_IN_GPU_TESTS and e not in NOT_ELEMENTWISE)
    assert not missing, ("entry points no element-wise test reaches (add a float64 or bit-exact test, or list them in "
                         "NOT_ELEMENTWISE with a reason): %s" % missing)
    stale = sorted(e for e in NOT_ELEMENTWISE if e in reach)
    assert not stale, "listed as without an element-wise test but reached by one: %s" % stale


def test_elementwise_reach_is_per_function():
    """Only the named functions of a mixed module count, with the module-level helpers they call; its other tests do not."""
    wrappers, callers = ops_wrappers(), package_callers()
    tree = ast.parse("from michigan_b200 import ops\n\n"
                     "def _run(x):\n    return ops.conv_thin(x)\n\n"
                     "def test_fp64():\n    _run(1)\n\n"
                     "def test_end_to_end():\n    ops.maxpool_mask(None, 3)\n")
    assert _test_module_reach(tree, wrappers, callers, _local_scope(tree, ["test_fp64"])) == {"mg_conv_thin"}
    assert _test_module_reach(tree, wrappers, callers, _local_scope(tree, ["test_end_to_end"])) == {"mg_maxpool_mask"}
    assert _test_module_reach(tree, wrappers, callers) == {"mg_conv_thin", "mg_maxpool_mask"}


def test_names_resolve_through_imports_only():
    """A local variable named like a package class or ops function credits nothing; the imported name does."""
    wrappers, callers = ops_wrappers(), package_callers()
    assert callers["SPADE"], "SPADE reaches entry points through its convs"
    local = ast.parse("SPADE = [1, 2]\nconv_thin = None\n\ndef test_x():\n    return SPADE, conv_thin\n")
    assert _test_module_reach(local, wrappers, callers) == set()
    imported = ast.parse("from michigan_b200.networks import SPADE\n\ndef test_x():\n    return SPADE\n")
    assert _test_module_reach(imported, wrappers, callers) == callers["SPADE"]
    getter = ast.parse("def _ops():\n    from michigan_b200 import ops\n    return ops\n\n"
                       "def test_x():\n    ops = _ops()\n    ops.conv_thin(None)\n    _ops().maxpool_mask(None, 3)\n")
    assert _test_module_reach(getter, wrappers, callers) == {"mg_conv_thin", "mg_maxpool_mask"}
    direct = ast.parse("def test_x(lib):\n    lib.load().mg_edge_weight(0)\n")
    assert _test_module_reach(direct, wrappers, callers) == {"mg_edge_weight"}


# ============================================================================================== backward stages
def backward_functions():
    """The hand-written backward functions of the package -> their AST nodes: the module-level `*_bwd` functions of
    networks/autograd.py, the `backward` of its autograd.Function classes ("Cls.backward") and every `backward_nhwc`
    method under networks/ ("Cls.backward_nhwc")."""
    net = os.path.join(PKG, "networks")
    _, tree = _parse(os.path.join(net, "autograd.py"))
    out = {}
    for node in tree.body:
        if isinstance(node, ast.FunctionDef) and node.name.endswith("_bwd"):
            out[node.name] = node
        elif isinstance(node, ast.ClassDef) and any(getattr(b, "attr", None) == "Function" for b in node.bases):
            out.update({node.name + ".backward": m for m in node.body if isinstance(m, ast.FunctionDef) and m.name == "backward"})
    for fn in sorted(os.listdir(net)):
        if fn.endswith(".py"):
            _, t = _parse(os.path.join(net, fn))
            for node in t.body:
                if isinstance(node, ast.ClassDef):
                    out.update({node.name + ".backward_nhwc": m for m in node.body
                                if isinstance(m, ast.FunctionDef) and m.name == "backward_nhwc"})
    return out


def backward_reach(tree, bwd):
    """The backward functions a module's code reaches: a function it names, a method whose class and name it both names,
    and, transitively, the backward functions their code names in turn."""
    def named(q, names):
        return all(part in names for part in q.split("."))
    reached, todo = set(), [q for q in bwd if named(q, _code_names(tree))]
    while todo:
        q = todo.pop()
        if q in reached:
            continue
        reached.add(q)
        inner = _code_names(bwd[q])
        todo.extend(r for r in bwd if r not in reached and named(r, inner))
    return reached


def test_backward_functions_are_found():
    bwd = backward_functions()
    assert {"block_bwd", "_spade_conv_bwd", "fc_bwd", "bg_bwd", "latent_bwd", "sn_conv_stack_bwd", "conv_encoder_bwd",
            "_d_scale_bwd", "_DiscriminatorFn.backward", "ImageEncoder3.backward_nhwc", "ImageEncoder2.backward_nhwc",
            "ImageEncoder.backward_nhwc"} <= set(bwd), sorted(bwd)


def test_every_backward_function_has_a_stage_test():
    bwd = backward_functions()
    _, tree = _parse(os.path.join(TESTS, BACKWARD_STAGES_MODULE))
    reached = backward_reach(tree, bwd)
    assert set(NOT_IN_BACKWARD_STAGES) <= set(bwd), sorted(set(NOT_IN_BACKWARD_STAGES) - set(bwd))
    missing = sorted(q for q in bwd if q not in reached and q not in NOT_IN_BACKWARD_STAGES)
    assert not missing, ("backward functions %s does not reach (add a stage test, or list them in NOT_IN_BACKWARD_STAGES "
                         "with a reason): %s" % (BACKWARD_STAGES_MODULE, missing))
    stale = sorted(q for q in NOT_IN_BACKWARD_STAGES if q in reached)
    assert not stale, "listed as left out but reached by %s: %s" % (BACKWARD_STAGES_MODULE, stale)


def test_backward_reach_follows_calls_and_needs_the_class():
    """A stage reached only through another backward function counts; a backward_nhwc counts only where its class is named
    too; a backward function the module stops calling is missing."""
    bwd = backward_functions()
    tree = ast.parse("from michigan_b200.networks import autograd, ImageEncoder2\n\n"
                     "def test_x(E, S):\n    autograd.block_bwd(None, None, S, None, None, None)\n"
                     "    assert isinstance(E, ImageEncoder2)\n    E.backward_nhwc(None, S, None)\n")
    reached = backward_reach(tree, bwd)
    assert {"block_bwd", "_spade_conv_bwd", "ImageEncoder2.backward_nhwc", "sn_conv_stack_bwd"} <= reached
    assert "ImageEncoder.backward_nhwc" not in reached and "bg_bwd" not in reached
    _, full = _parse(os.path.join(TESTS, BACKWARD_STAGES_MODULE))
    src = ast.unparse(full).replace("autograd.bg_bwd(", "autograd.block_bwd(")
    assert "bg_bwd" not in backward_reach(ast.parse(src), bwd)
