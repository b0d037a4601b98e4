"""TEST / BASELINE INFRASTRUCTURE: build the reference's own COVID-19 CUDA kernels for sm_90a.

    python oracle/build_ref_covid.py          ->  oracle/_ref/libref_covid_cuda.so   (git-ignored)

The kernels are compiled FROM THE SOURCES WHERE THEY LIE under /root/reference (scenarios/covid19/covid19_build.cu, which
includes components/covid19_components_step.cu and scenarios/covid19/covid19_env_step.cu); nothing of the reference is
copied into the repository.  oracle/ref_covid_launcher.cu (ours) adds the host-side launch sequence that the reference
keeps in Python on top of WarpDrive/PyCUDA.  Without the reference sources this is a no-op and the prebuilt
library, if any, is used as it is.  Flags: the reference is built the way WarpDrive builds it (nvcc defaults: -O3,
fused multiply-add allowed) - it is the baseline, it gets its own best settings.
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
REF_BUILD_CU = "/root/reference/ai_economist/foundation/scenarios/covid19/covid19_build.cu"
OUT_DIR = os.path.join(HERE, "_ref")
LIB = os.path.join(OUT_DIR, "libref_covid_cuda.so")
LAUNCHER = os.path.join(HERE, "ref_covid_launcher.cu")


def available():
    return os.path.exists(LIB)


def build(force=False, verbose=False):
    """Returns the library path, or None when neither the reference sources nor a prebuilt library exist."""
    if not os.path.exists(REF_BUILD_CU):
        return LIB if available() else None
    deps = [LAUNCHER, REF_BUILD_CU, os.path.join(os.path.dirname(REF_BUILD_CU), "covid19_env_step.cu"),
            "/root/reference/ai_economist/foundation/components/covid19_components_step.cu"]
    if not force and available() and os.path.getmtime(LIB) >= max(os.path.getmtime(d) for d in deps):
        return LIB
    os.makedirs(OUT_DIR, exist_ok=True)
    cmd = [os.environ.get("NVCC", "nvcc"), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-shared",
           "-Xcompiler", "-fPIC", '-DREF_COVID_BUILD_CU="%s"' % REF_BUILD_CU, "-o", LIB, LAUNCHER]
    if verbose:
        cmd += ["-Xptxas", "-v"]
    subprocess.check_call(cmd)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
