"""CPU oracle of the skeletal-animation entry points — TEST INFRASTRUCTURE, like the rest of this package.

libr3_oracle_anim.so (r3_oracle_anim.c) links libr3_oracle.so: loading it gives one handle through which every r3o_ entry point
resolves, so a rend3_b200.backend.Backend bound to it is the full oracle plus r3o_set_animations ... r3o_readback_joint_matrices."""
import ctypes
import os
import subprocess

from . import _DIR
from . import build as build_oracle

LIB_PATH = os.path.join(_DIR, "libr3_oracle_anim.so")
# the flags of oracle/Makefile: strict IEEE f32, no contraction
CFLAGS = ["-O3", "-mavx2", "-std=gnu11", "-fPIC", "-fopenmp", "-ffp-contract=off", "-fno-fast-math", "-fvisibility=hidden",
          "-Wall", "-Wextra", "-Wno-unused-parameter"]


def build(force: bool = False) -> str:
    base = build_oracle()
    srcs = [os.path.join(_DIR, "r3_oracle_anim.c"), os.path.join(_DIR, "r3_oracle.h"), base, __file__]
    srcs += [os.path.join(_DIR, "..", "include", f) for f in ("r3_layouts.h", "rend3_b200.h", "r3_anim_check.h")]
    stale = force or not os.path.exists(LIB_PATH) or any(os.path.exists(s) and os.path.getmtime(s) > os.path.getmtime(LIB_PATH) for s in srcs)
    if stale:
        cc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc"
        cmd = [cc, *CFLAGS, "-shared", "-o", LIB_PATH, os.path.join(_DIR, "r3_oracle_anim.c"), "-L", _DIR, "-l:libr3_oracle.so",
               "-Wl,-rpath,$ORIGIN", "-lm", "-lpthread"]
        try:
            subprocess.run(cmd, check=True, capture_output=True, text=True)
        except (subprocess.CalledProcessError, FileNotFoundError) as e:  # keep a prebuilt .so usable on boxes without gcc
            if not os.path.exists(LIB_PATH):
                raise RuntimeError(f"animation oracle build failed: {getattr(e, 'stderr', e)}")
    return LIB_PATH


def load_anim_oracle_backend():
    """A Backend over the oracle with the animation entry points; closing it also drops the context's animation state."""
    from rend3_b200.backend import Backend

    class AnimOracleBackend(Backend):
        def close(self):
            if self.ctx:
                self.lib.r3o_anim_release(self.ctx)
            super().close()

    return AnimOracleBackend(ctypes.CDLL(build()), "r3o_", 0)
