"""Every kernel entry point of scail_b200.ops is checked at the shapes the product launches.

The launch-shape harnesses (test_dit_launch_shapes_gpu, test_cp_launch_shapes_gpu, test_vae_launch_shapes_gpu and
test_dit_int8_b1_launch_shapes_gpu) record the entry points named in their OPS tuples while a real workload runs and re-check
every distinct launch against fp32.  An entry point that enters none of those tuples is never checked that way: the INT8
Q·Kᵀ mode went without it for a release.  So each function of ops.py that calls into the library must appear in one of the
tuples or in ELSEWHERE below, which names the test that checks it at the production latents and why that test suffices.
Everything is read with ast: no GPU module is imported."""
import ast
import os

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TESTS = os.path.join(ROOT, "tests")
HARNESSES = ("test_dit_launch_shapes_gpu.py", "test_cp_launch_shapes_gpu.py", "test_vae_launch_shapes_gpu.py",
             "test_dit_int8_b1_launch_shapes_gpu.py")
_LATENTS = "at the 21x64x64, 21x60x104 and 21x64x112 latents"

# entry point -> (file::test that checks it at the production latents, why that is enough)
ELSEWHERE = {
    "cfg_cache_delta": ("test_cfg_cache_gpu.py::test_delta_kernel",
                        f"elementwise over the CFG pair: sums against fp64 and delta bit for bit {_LATENTS}"),
    "cfg_euler_cached_": ("test_cfg_cache_gpu.py::test_cached_euler_kernel",
                          f"elementwise on the latent: bit for bit its restatement {_LATENTS}"),
    "unipc_step_cached_": ("test_cfg_cache_gpu.py::test_cached_unipc_kernel",
                           f"elementwise on the latent and its slots: bit for bit its restatement {_LATENTS}"),
    "cfg_cache_delta_forecast": ("test_cfg_cache_forecast_gpu.py::test_delta_forecast_kernel",
                                 f"elementwise with slot and coefficient patterns: against fp64 and bit for bit {_LATENTS}"),
    "cfg_euler_cached_forecast_": ("test_cfg_cache_forecast_gpu.py::test_cached_euler_forecast_kernel",
                                   f"elementwise on the latent: bit for bit its restatement {_LATENTS}"),
    "unipc_step_cached_forecast_": ("test_cfg_cache_forecast_gpu.py::test_cached_unipc_forecast_kernel",
                                    f"elementwise on the latent and its slots: bit for bit its restatement {_LATENTS}"),
    "cfg_zero_scale": ("test_cfg_zero_gpu.py::test_scale_pair",
                       f"a reduction over the CFG pair against fp64 {_LATENTS}; cached and forecast forms in test_scale_cached "
                       "and test_scale_forecast"),
    "apg_reduce": ("test_apg_gpu.py::test_kernels_against_the_oracle",
                   f"per-frame reductions against the fp64 oracle in the pair, cached and forecast forms {_LATENTS}"),
    "apg_finish": ("test_apg_gpu.py::test_kernels_against_the_oracle",
                   f"the fp64 finish of those reductions, against the oracle {_LATENTS}"),
    "apg_update_": ("test_apg_gpu.py::test_kernels_against_the_oracle",
                    f"elementwise update against the oracle {_LATENTS}"),
    "unipc_step_dpred_": ("test_apg_gpu.py::test_unipc_data_prediction_kernel",
                          f"elementwise on the latent and its slots: bit for bit its restatement {_LATENTS}"),
    "vae_latent_to_cl": ("test_vae_gpu.py::test_latent_to_cl_at_the_production_latents",
                         "elementwise: bit for bit one division and one addition at the 21-frame latents of all three sizes"),
}


def lib_entry_points(source):
    """Top-level functions of `source` (ops.py text) whose body uses the name _lib."""
    return sorted(n.name for n in ast.parse(source).body if isinstance(n, ast.FunctionDef)
                  and any(isinstance(x, ast.Name) and x.id == "_lib" for x in ast.walk(n)))


def _assignments(path):
    """{name: expression node} of the module-level assignments of one test file, and {name: module} of its
    `from <module> import name` lines."""
    tree = ast.parse(open(path).read())
    names, imported = {}, {}
    for n in tree.body:
        if isinstance(n, ast.Assign) and len(n.targets) == 1 and isinstance(n.targets[0], ast.Name):
            names[n.targets[0].id] = n.value
        elif isinstance(n, ast.ImportFrom) and n.module:
            for a in n.names:
                imported[a.asname or a.name] = n.module
    return names, imported


def _resolve(expr, path, seen=()):
    """The strings of a tuple expression: literal tuples, names bound in the file or imported from another test file, and
    sums of those (CP_OPS = OPS + (...))."""
    if isinstance(expr, ast.Tuple):
        assert all(isinstance(e, ast.Constant) and isinstance(e.value, str) for e in expr.elts), ast.dump(expr)
        return tuple(e.value for e in expr.elts)
    if isinstance(expr, ast.BinOp) and isinstance(expr.op, ast.Add):
        return _resolve(expr.left, path, seen) + _resolve(expr.right, path, seen)
    if isinstance(expr, ast.Name):
        key = (path, expr.id)
        assert key not in seen, f"a cycle through {expr.id}"
        names, imported = _assignments(path)
        if expr.id in names:
            return _resolve(names[expr.id], path, seen + (key,))
        if expr.id in imported:
            other = os.path.join(os.path.dirname(path), imported[expr.id] + ".py")
            return _resolve(ast.Name(id=expr.id), other, seen + (key,))
    raise AssertionError(f"{path}: cannot resolve {ast.dump(expr)}")


def recorded_ops(path):
    """Every entry point named by a module-level *OPS tuple of one harness file."""
    names, _ = _assignments(path)
    return {op for name, expr in names.items() if name.endswith("OPS") for op in _resolve(expr, path)}


def unchecked(ops_source, recorded, elsewhere):
    """Entry points of ops_source in neither the recorded set nor the table."""
    return [f for f in lib_entry_points(ops_source) if f not in recorded and f not in elsewhere]


def _ops_source():
    return open(os.path.join(ROOT, "scail_b200", "ops.py")).read()


def _all_recorded():
    out = set()
    for h in HARNESSES:
        out |= recorded_ops(os.path.join(TESTS, h))
    return out


def test_every_entry_point_is_recorded_or_points_to_its_test():
    recorded = _all_recorded()
    missing = unchecked(_ops_source(), recorded, ELSEWHERE)
    assert not missing, (f"ops.py entry points in no launch-shape OPS tuple and not in ELSEWHERE: {missing}; record them in a "
                         "harness or name the test that checks them at the production shapes")
    entry = set(lib_entry_points(_ops_source()))
    stale = sorted(set(ELSEWHERE) - entry)
    assert not stale, f"ELSEWHERE names functions ops.py no longer has or that no longer launch: {stale}"
    both = sorted(set(ELSEWHERE) & recorded)
    assert not both, f"recorded by a harness and also listed in ELSEWHERE: {both}"
    assert not recorded - entry, f"OPS tuples name what ops.py does not launch: {sorted(recorded - entry)}"


@pytest.mark.parametrize("name", sorted(ELSEWHERE))
def test_each_table_entry_names_a_test_that_exists(name):
    where, why = ELSEWHERE[name]
    assert why.strip()
    file, test = where.split("::")
    tree = ast.parse(open(os.path.join(TESTS, file)).read())
    tests = {n.name: n for n in tree.body if isinstance(n, ast.FunctionDef)}
    assert test in tests, f"{where} does not exist"
    calls = {x.attr for x in ast.walk(tests[test]) if isinstance(x, ast.Attribute) and x.value.__class__ is ast.Name
             and x.value.id == "ops"}
    assert name in calls, f"{where} does not call ops.{name}"


def test_the_cp_sum_and_the_int8_tuples_resolve():
    cp = recorded_ops(os.path.join(TESTS, "test_cp_launch_shapes_gpu.py"))
    dit = recorded_ops(os.path.join(TESTS, "test_dit_launch_shapes_gpu.py"))
    assert dit < cp and {"attention_partial", "attention_merge"} <= cp
    int8 = recorded_ops(os.path.join(TESTS, "test_dit_int8_b1_launch_shapes_gpu.py"))
    assert dit < int8 and {"rmsnorm_rope_int8q", "quant_k_int8", "attention_int8qk"} <= int8


def test_the_checker_reports_an_extra_entry_point():
    extra = _ops_source() + '\n\ndef brand_new_kernel(x):\n    _lib.check(_lib.lib().scail_brand_new(_ptr(x), _stream()), "n")\n'
    assert unchecked(extra, _all_recorded(), ELSEWHERE) == ["brand_new_kernel"]
    # a helper that does not call into the library is not an entry point
    helper = _ops_source() + "\n\ndef brand_new_helper(x):\n    return x\n"
    assert unchecked(helper, _all_recorded(), ELSEWHERE) == []
    # and an entry point dropped from the tuples is reported
    assert unchecked(_ops_source(), _all_recorded() - {"quant_k_int8"}, ELSEWHERE) == ["quant_k_int8"]
