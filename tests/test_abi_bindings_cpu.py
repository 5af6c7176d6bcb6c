"""CPU: the Python side of the C ABI agrees with include/tsc.h and include/tsc_learn.h.

- Prototypes: after loading, every declared function carries the header's parameter count and the ctypes types the
  header's C types map to.
- Call sites: every literal call of a declared function in the package, scripts, tests and oracle passes the
  prototype's number of arguments (ctypes raises for too few, but passes surplus arguments along silently) and every
  explicit ctypes wrapper matches its parameter's C type.
- Struct layout: the ctypes mirrors CNet, CCfg, CDims and CQDims have the header structs' fields, in order, at the
  offsets and sizes the system C compiler gives them."""
import ast
import ctypes as C
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADERS = [os.path.join(ROOT, "include", h) for h in ("tsc.h", "tsc_learn.h")]
SCALARS = {"int32_t": "c_int32", "int64_t": "c_int64", "uint64_t": "c_uint64", "float": "c_float"}
WRAPPERS = {"c_int32", "c_int64", "c_uint64", "c_float", "c_void_p"}


def _source(path):
    return re.sub(r"/\*.*?\*/", "", open(path).read(), flags=re.S)


def _c_type(decl):
    """ctypes name of one header parameter: 'c_void_p' for any pointer, else its scalar type."""
    if "*" in decl:
        return "c_void_p"
    return SCALARS[decl.replace("const ", "").split()[0]]


def _prototypes():
    """{name: (return type, [ctypes name of each parameter])} as the headers declare them."""
    protos = {}
    for path in HEADERS:
        for ret, name, params in re.findall(r"^\s*(int|const char\*)\s+(tscl?_[a-z0-9_]+)\s*\(([^)]*)\)", _source(path),
                                            flags=re.M):
            params = [p.strip() for p in " ".join(params.split()).split(",")]
            protos[name] = (ret, [] if params in ([""], ["void"]) else [_c_type(p) for p in params])
    return protos


PROTOS = _prototypes()


def test_loaded_functions_carry_the_header_prototypes():
    from deeprl_signal_control_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        _lib.build_native()
    lib = _lib.lib()
    assert len(PROTOS) >= 68 and set(PROTOS) == set(_lib.SYMBOLS)
    assert len(PROTOS["tscl_policy_step_v2r"][1]) == 27 and PROTOS["tsc_last_error"] == ("const char*", [])
    for name, (ret, params) in PROTOS.items():
        fn = getattr(lib, name)
        assert fn.restype is (C.c_char_p if ret == "const char*" else C.c_int), name
        assert fn.argtypes is not None and len(fn.argtypes) == len(params), name
        assert list(fn.argtypes) == [getattr(C, p) for p in params], name


def _python_files():
    for top in ("deeprl_signal_control_b200", "scripts", "tests", "oracle"):
        for dp, dirs, fs in os.walk(os.path.join(ROOT, top)):
            dirs[:] = [d for d in dirs if d != "__pycache__"]
            yield from (os.path.join(dp, f) for f in sorted(fs) if f.endswith(".py"))
    yield os.path.join(ROOT, "__graft_entry__.py")


def _declared_calls(tree):
    """(name, positional argument nodes, keywords, node) of every `<x>.<declared>(...)` and `_call("<declared>", ...)`."""
    for n in ast.walk(tree):
        if not isinstance(n, ast.Call):
            continue
        if isinstance(n.func, ast.Attribute) and n.func.attr in PROTOS:
            yield n.func.attr, n.args, n.keywords, n
        elif (isinstance(n.func, ast.Name) and n.func.id == "_call" and n.args
              and isinstance(n.args[0], ast.Constant) and n.args[0].value in PROTOS):
            yield n.args[0].value, n.args[1:], n.keywords, n


def _wrapper(arg):
    """'c_int32' etc. for an argument written as `C.c_int32(...)` / `ctypes.c_int32(...)`, else None."""
    if (isinstance(arg, ast.Call) and isinstance(arg.func, ast.Attribute) and arg.func.attr in WRAPPERS
            and isinstance(arg.func.value, ast.Name) and arg.func.value.id in ("C", "ctypes")):
        return arg.func.attr
    return None


def call_site_errors(paths):
    errors, n_calls = [], 0
    for path in paths:
        tree = ast.parse(open(path).read(), filename=path)
        for name, args, keywords, node in _declared_calls(tree):
            n_calls += 1
            where = "%s:%d %s" % (os.path.relpath(path, ROOT), node.lineno, name)
            want = PROTOS[name][1]
            starred = [i for i, a in enumerate(args) if isinstance(a, ast.Starred)]
            fixed = len(args) - len(starred)
            if keywords:
                errors.append("%s: keyword arguments" % where)
            if not starred and fixed != len(want):
                errors.append("%s: %d arguments, the prototype has %d" % (where, fixed, len(want)))
            if starred and fixed > len(want):
                errors.append("%s: %d fixed arguments besides *args, the prototype has %d" % (where, fixed, len(want)))
            # positions are known up to the first *args
            for i, a in enumerate(args[:starred[0] if starred else len(args)]):
                w = _wrapper(a)
                if w is not None and i < len(want) and w != want[i]:
                    errors.append("%s: argument %d is C.%s, the header declares %s" % (where, i, w, want[i]))
    return errors, n_calls


def test_call_sites_match_the_prototypes():
    errors, n_calls = call_site_errors(list(_python_files()))
    assert n_calls > 100                # the package, scripts and tests call the library in ~190 places
    assert not errors, "\n".join(errors)


def test_call_site_check_catches_each_kind_of_mismatch(tmp_path):
    bad = tmp_path / "bad.py"
    bad.write_text("lib.tsc_set_train_mode(h)\n"                          # one argument short
                   "lib.tsc_set_train_mode(h, 1, 2)\n"                    # one argument too many
                   "lib.tsc_set_record(h, on=1)\n"                        # a keyword
                   "lib.tscl_dx_tc(h, a, b, c, C.c_int32(M), s)\n"        # int64_t wrapped as int32
                   "lib.tscl_dx_tc(*args, h, a, b, c, M, s)\n"            # too many beside *args
                   "_call('tsc_mean_live', h)\n")                         # one argument short through _call
    errors, n_calls = call_site_errors([str(bad)])
    assert n_calls == 6 and len(errors) == 6, errors


def _struct_fields(body):
    """Field names of a C struct body, in order (comma lists included)."""
    names = []
    for decl in body.split(";"):
        decl = decl.strip()
        if decl:
            head, *rest = decl.split(",")
            names += [re.findall(r"\w+", head)[-1]] + [re.findall(r"\w+", r)[-1] for r in rest]
    return names


def test_struct_mirrors_match_the_headers(tmp_path):
    from deeprl_signal_control_b200.agents.layout import CDims, CQDims
    from deeprl_signal_control_b200.net.tables import CCfg, CNet
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no C compiler on the path")
    mirrors = {"tsc_net": CNet, "tsc_cfg": CCfg, "tscl_dims": CDims, "tscl_qdims": CQDims}
    src = "".join(_source(h) for h in HEADERS)
    fields = {name: _struct_fields(body) for body, name in
              re.findall(r"typedef struct \w+ \{(.*?)\} (\w+);", src, flags=re.S)}
    assert set(mirrors) <= set(fields)
    probe = ['#include <stddef.h>\n#include <stdio.h>\n#include "tsc.h"\n#include "tsc_learn.h"\nint main(void) {\n']
    for s in mirrors:
        probe.append('  printf("%s %%zu\\n", sizeof(%s));\n' % (s, s))
        probe += ['  printf("%s.%s %%zu %%zu\\n", offsetof(%s, %s), sizeof(((%s*)0)->%s));\n' % (s, f, s, f, s, f)
                  for f in fields[s]]
    (tmp_path / "probe.c").write_text("".join(probe) + "  return 0;\n}\n")
    exe = str(tmp_path / "probe")
    subprocess.run([cc, "-I", os.path.join(ROOT, "include"), str(tmp_path / "probe.c"), "-o", exe], check=True)
    c_layout = {}
    for line in subprocess.run([exe], capture_output=True, text=True, check=True).stdout.splitlines():
        key, *vals = line.split()
        c_layout[key] = tuple(int(v) for v in vals)
    for s, mirror in mirrors.items():
        assert [f[0] for f in mirror._fields_] == fields[s], s
        assert C.sizeof(mirror) == c_layout[s][0], s
        for f in fields[s]:
            got = getattr(mirror, f)
            assert (got.offset, got.size) == c_layout["%s.%s" % (s, f)], (s, f)
