"""CPU: what the compiler makes of the GEMM kernel's consumer mainloop (csrc/gemm_v3.cu), read from ptxas and the SASS.

Each pipeline stage must be one wgmma chain: one WARPGROUP.ARRIVE, then every HGMMA of the stage, closed by the last one's
gsb0.  ptxas breaks a chain into fenced groups (and says so with C7519 / C7510) when accumulator registers are touched between
wgmmas; the groups then run one after the other with the tensor pipe drained in between."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "vehicle-cv-adas_b200", "csrc")
CUDA_BIN = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin")


def _tool(name):
    p = shutil.which(name) or os.path.join(CUDA_BIN, name)
    return p if os.path.isfile(p) and os.access(p, os.X_OK) else None


NVCC, CUOBJDUMP = _tool("nvcc"), _tool("cuobjdump")
pytestmark = pytest.mark.skipif(NVCC is None or CUOBJDUMP is None, reason="needs nvcc and cuobjdump")

K128 = "_ZN4adas19conv_gemm_v3_kernelILi128ELb0ELb0EEEv14CUtensorMap_stS1_NS_6GemmV3E"


def _make_flags():
    """ARCH, CXXFLAGS and gemm_v3.o's SPLIT of csrc/Makefile: the test compiles what the build compiles."""
    mk = open(os.path.join(CSRC, "Makefile")).read()
    flags = []
    for var in ("ARCH", "CXXFLAGS"):
        flags += re.search(rf"^{var} := (.*)$", mk, re.M).group(1).split()
    flags += re.search(r"^gemm_v3\.o: SPLIT := (.*)$", mk, re.M).group(1).split()
    return flags


@pytest.fixture(scope="module")
def gemm_build(tmp_path_factory):
    out = tmp_path_factory.mktemp("gemm_codegen")
    obj = str(out / "gemm_v3.o")
    r = subprocess.run([NVCC, *_make_flags(), "-Xptxas", "-v", "-c", os.path.join(CSRC, "gemm_v3.cu"), "-o", obj],
                       cwd=CSRC, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    return r.stdout + r.stderr, obj


def _sass(obj, fn):
    r = subprocess.run([CUOBJDUMP, "-sass", "-fun", fn, obj], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    ins = re.findall(r"/\*[0-9a-f]{4,}\*/\s+(.*?)\s*;", r.stdout)
    assert ins, f"no SASS for {fn}"
    return ins


def _chains(ins):
    """Every run from a WARPGROUP.ARRIVE to the HGMMA that closes its group (gsb0): (instructions, index of the ARRIVE)."""
    chains, i = [], 0
    while i < len(ins):
        if ins[i].startswith("WARPGROUP.ARRIVE"):
            j = i + 1
            while j < len(ins) and not ("HGMMA" in ins[j] and "gsb0" in ins[j]):
                j += 1
            assert j < len(ins), "a WARPGROUP.ARRIVE without a closing HGMMA"
            chains.append(ins[i:j + 1])
            i = j + 1
        else:
            i += 1
    return chains


def test_no_injected_fences(gemm_build):
    log, _ = gemm_build
    entries = re.findall(r"Compiling entry function '(_ZN4adas19conv_gemm_v3_kernel\w+)'", log)
    assert len(entries) == 38, f"expected the 38 conv_gemm_v3_kernel instantiations, ptxas compiled {len(entries)}"
    bad = [ln for ln in log.splitlines() if re.search(r"C75(19|10)", ln) and "conv_gemm_v3_kernel" in ln]
    assert not bad, f"{len(bad)} injected-fence / serialised-wgmma warnings, e.g.\n" + "\n".join(bad[:5])


def test_bn128_one_chain_per_stage(gemm_build):
    _, obj = gemm_build
    ins = _sass(obj, K128)
    chains = _chains(ins)
    # BN 128 holds four specialised mainloops -- sub-tiles MT = 1, 2 x taps per stage 1, 3 -- each stage issuing
    # TPS * MT * (BK / 16 = 4) wgmmas of 64x128x16
    assert sum(x.startswith("WARPGROUP.ARRIVE") for x in ins) == len(chains) == 4, [len(c) for c in chains]
    counts = sorted(sum("HGMMA" in x for x in c) for c in chains)
    assert counts == [4, 8, 12, 24], counts
    for c in chains:
        hg = [x for x in c if "HGMMA" in x]
        assert all(x.startswith("HGMMA.64x128x16.F32 ") for x in hg), hg
        assert sum("gsb0" in x for x in hg) == 1, "a stage's chain is closed more than once"
        assert not [x for x in c if re.search(r"\b(LDL|STL)\b", x)], "spill access inside a wgmma chain"
    dummy = [x for x in ins if re.match(r"HGMMA\.\S+ RZ,", x)]
    assert not dummy, f"dummy HGMMA commit: {dummy}"
