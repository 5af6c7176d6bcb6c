"""Golden text of the fixed-time programs the REFERENCE's scenario generators write (exp.tll.xml): `output_tls` of
large_grid/data/build_file.py and small_grid/data/build_file.py, called with the tlLogic / phase templates their main()
passes.  net/large_grid.py and net/small_grid.py restate these programs as data; tests/test_fixedtime_cpu.py pins them
against this file.     Run: python tests/golden/gen_tls_golden.py
"""
import importlib.util
import json
import os

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("REFERENCE_ROOT", "/root/reference")
TLS = '  <tlLogic id="%s" programID="0" offset="0" type="static">\n'     # build_file.py:main, both scenarios
PHASE = '    <phase duration="%d" state="%s"/>\n'


def _generator(scenario):
    spec = importlib.util.spec_from_file_location("build_file_" + scenario,
                                                  os.path.join(REF, scenario, "data", "build_file.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


if __name__ == "__main__":
    out = {s: _generator(s).output_tls(TLS, PHASE) for s in ("large_grid", "small_grid")}
    with open(os.path.join(HERE, "tls_programs.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")
