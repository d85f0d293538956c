"""TEST INFRASTRUCTURE -- recipe for oracle/_ref/pyref with the reference's particle optimizer added: the byte-code build of
oracle/build_pyref.py (the call sites of the kernel backends and the L-BFGS optimizer), plus curobo._src.optim.particle.mppi and
its import closure, compiled from the sources where they lie under /root/reference.  tests/test_gpu_mppi.py drives the
reference's own MPPI class over B200RobotRollout from this build on the GPU box, where /root/reference does not exist.  No
reference source is copied into the repository.

    python oracle/build_pyref_particle.py   # needs /root/reference; writes oracle/_ref/pyref/ + MANIFEST.json
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import build_pyref  # noqa: E402

PARTICLE_CALL_SITES = ["curobo._src.optim.particle.mppi"]


def build(verbose: bool = False) -> str:
    build_pyref.CALL_SITES = build_pyref.CALL_SITES + PARTICLE_CALL_SITES
    return build_pyref.build(verbose)


if __name__ == "__main__":
    print(build(verbose=True))
