"""Record the parameter names (in order) and defaults of the reference's legacy trajectory launchers -- the POSITION (clique)
and ACCELERATION control spaces -- so that tests/test_position_clique_cpu.py can hold curobo_b200/backends/trajectory.py to
them without the reference tree present.  Same record format as make_signature_golden.py.
Needs /root/reference (authoring container only):  python tests/golden/make_legacy_signature_golden.py"""
import inspect
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import _reference_under_shim as R  # noqa: E402

R.prepare()
NAMES = ["launch_differentiation_position_forward_kernel", "launch_differentiation_position_backward_kernel",
         "launch_integration_acceleration_kernel"]
m = R.ref("curobo._src.curobolib.backends.cuda_core_backend.trajectory")
out = {}
for n in NAMES:
    fn = getattr(m, n)
    sig = inspect.signature(fn)
    out[f"trajectory.{n}"] = {"file": os.path.relpath(inspect.getsourcefile(fn), "/root/reference"),
                              "line": inspect.getsourcelines(fn)[1],
                              "params": [p.name for p in sig.parameters.values()],
                              "defaults": {p.name: repr(p.default) for p in sig.parameters.values()
                                           if p.default is not inspect.Parameter.empty}}
path = os.path.join(HERE, "reference_legacy_trajectory_signatures.json")
json.dump(out, open(path, "w"), indent=1, sort_keys=True)
print(f"wrote {path}: {len(out)} launchers")
