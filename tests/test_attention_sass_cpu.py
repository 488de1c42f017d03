"""CPU: the softmax stage of the attention kernels GPT-2 (C2) launches is straight-line code in the built library.

Between the wait on the S = Q K^T accumulator and the next wgmma (P V in the forward, dS K in the dQ kernel) the SASS of
attn_fwd_kernel<64, false, false, 0> and attn_bwd_dq_kernel<64, false, false, 0> must hold no BSSY / BSYNC
(reconvergence points of a divergent branch) and at most one branch: the warp-uniform one that skips the mask selects on
an unmasked step. The retry branch of an mbarrier try-wait (the wait for V in the forward) is not counted. Per-score
branches here cost 64 taken branches and reconvergence points per warp per key step and stop the scheduler from
interleaving the independent per-score work. Skipped when cuobjdump or the built library is missing."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "fengshen-lm_b200", "fsb200", "lib", "libfsb200.so")

KERNELS = {
    "attn_fwd_kernel<64,false,false,0>":
        "_ZN3fsb15attn_fwd_kernelILi64ELb0ELb0ELi0EEEv14CUtensorMap_stS1_S1_NS_12AttFwdParamsE",
    "attn_bwd_dq_kernel<64,false,false,0>":
        "_ZN3fsb18attn_bwd_dq_kernelILi64ELb0ELb0ELi0EEEv14CUtensorMap_stS1_S1_S1_NS_12AttBwdParamsE",
}


def _cuobjdump():
    exe = shutil.which("cuobjdump")
    if exe is None:
        cand = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")
        exe = cand if os.access(cand, os.X_OK) else None
    return exe


def _sass(exe, mangled):
    """The kernel's instructions, in address order, without addresses and encodings."""
    out = subprocess.run([exe, "-sass", "-fun", mangled, LIB], capture_output=True, text=True, check=True).stdout
    return [m.group(1).strip() for m in re.finditer(r"/\*[0-9a-f]{4,}\*/\s+([^;]*);", out)]


def _softmax_window(ins):
    """From the first wgmma wait after the first HGMMA (the wait on S) up to the next HGMMA."""
    first = next(i for i, s in enumerate(ins) if s.startswith("HGMMA"))
    wait = next(i for i in range(first, len(ins)) if ins[i].startswith("WARPGROUP.DEPBAR"))
    nxt = next(i for i in range(wait, len(ins)) if ins[i].startswith("HGMMA"))
    return ins[wait:nxt]


def _barrier_retry(win, opcode, k):
    """Branch k is predicated on the result of an mbarrier try-wait (its predicate was last written by SYNCS.PHASECHK)."""
    m = re.match(r"@!?(P\d)\s", win[k])
    if m is None:
        return False
    for j in range(k - 1, -1, -1):
        dst = win[j].split(None, 2)[1:2] if not win[j].startswith("@") else win[j].split(None, 3)[2:3]
        if dst and dst[0].rstrip(",") == m.group(1):
            return opcode[j].startswith("SYNCS.PHASECHK")
    return False


@pytest.mark.parametrize("name", sorted(KERNELS))
def test_softmax_stage_is_branch_free(name):
    exe = _cuobjdump()
    if exe is None:
        pytest.skip("cuobjdump not found")
    if not os.path.exists(LIB):
        pytest.skip("libfsb200.so not built")
    ins = _sass(exe, KERNELS[name])
    assert ins, f"{name} not found in {LIB}"
    win = _softmax_window(ins)
    opcode = [re.sub(r"^@!?U?P\w+\s+", "", s).split()[0] for s in win]
    recon = [s for s, op in zip(win, opcode) if op in ("BSSY", "BSYNC")]
    assert not recon, f"{name}: {len(recon)} BSSY/BSYNC between the wait on S and the next wgmma"
    branches = [s for k, (s, op) in enumerate(zip(win, opcode)) if op.startswith("BRA") and not _barrier_retry(win, opcode, k)]
    assert len(branches) <= 1, f"{name}: {len(branches)} branches between the wait on S and the next wgmma: {branches}"
