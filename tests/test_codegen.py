"""CPU: properties of the generated sm_90a code that the kernel's speed depends on (checked on the built library).

poa_simt.cuh explains the first one: ptxas gives EVERY warp collective of the module a "BRA.DIV -> WARPSYNC.COLLECTIVE"
slow path (and BSSY/BSYNC brackets, and the registers to feed them: +43 % instructions) as soon as it cannot prove the
control flow around ONE of them warp-uniform.  The property is global and fragile (a by-reference parameter, one
un-laundered shuffle result steering a loop), so it is pinned here."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "racon_gpu_b200", "libb200poa.so")


@pytest.fixture(scope="module")
def sass():
    if not shutil.which("cuobjdump"):
        pytest.skip("cuobjdump not available")
    from racon_gpu_b200 import api
    api.load_library()  # builds if needed
    out = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True, check=True).stdout
    assert "poa_window_kernel" in out
    # the POA kernel's own code: the library also holds the overlap aligner's kernels (csrc/b200aln.cu, another module --
    # its team kernel spins on progress words, which is lane-dependent control flow by construction)
    start = out.index("poa_window_kernel")
    nxt = out.find("Function :", start)
    return out[start:nxt if nxt > 0 else len(out)]


def test_no_divergence_slow_paths_anywhere_in_the_kernel(sass):
    assert sass.count("BRA.DIV") == 0, "a warp collective is reachable from control flow ptxas cannot prove uniform"
    assert sass.count("WARPSYNC.COLLECTIVE") == 0


def test_the_fill_uses_the_packed_int16_pipeline_and_async_copies(sass):
    """The DP fill's cells are packed int16 pairs (VIADDMNMX.S16x2 / VIMNMX3.S16x2: Hopper's DPX instructions), the
    traceback tile arrives by asynchronous global->shared copies (LDGSTS), warp reductions are single REDUX
    instructions, results leave with streaming stores."""
    for op in ("VIADDMNMX.S16x2", "VIMNMX3.S16x2", "LDGSTS", "REDUX", "STG.E.EF.128"):
        assert op in sass, op
    n_instr = len(re.findall(r"^\s+/\*[0-9a-f]{4,6}\*/", sass, flags=re.M))
    # sm_90a at 20 blocks/SM: 14 536 instructions, about 1 900 of them local-memory moves; divergence slow paths add ~40 %
    assert n_instr < 14650, f"kernel grew to {n_instr} instructions: check for divergence fallbacks or unrolling"


def _uniform_regs_read_by_async_copies_are_written(sass):
    written = set(re.findall(r"^\s+/\*[0-9a-f]{4,6}\*/\s+(?:@!?U?P[T0-9]\s+)?[A-Z][A-Z0-9_.]*\s+(UR\d+)\b", sass, flags=re.M))
    used = set()
    for line in re.findall(r"LDGSTS[^;]*;", sass):
        used.update(re.findall(r"\b(UR\d+)\b", line))
    return used, written


def test_every_async_copy_reads_uniform_registers_the_kernel_writes(sass):
    """Each LDGSTS of the traceback tile takes its memory descriptor (and possibly an address base) from uniform
    registers; ptxas 12.9 compiles the L2-cache-hinted form into copies reading UR0 / UR1 that nothing writes, which the
    H100 reports as an illegal instruction at the first tile load (poa_core.cuh: tile_copy16, DESIGN §10)."""
    used, written = _uniform_regs_read_by_async_copies_are_written(sass)
    assert used and used <= written, sorted(used - written)


def _function_section(out, name):
    import re as _re
    m = _re.search(r"Function : \S*" + name + r"\S*", out)
    assert m, name
    nxt = out.find("Function :", m.end())
    return out[m.start():nxt if nxt > 0 else len(out)]


def test_aligner_step_loop_keeps_its_shape():
    """csrc/aln_core.cuh myers_pass: the one-warp split kernel's wavefront runs 16 steps to a group (16 SHFL.UP in the
    unrolled loop + 1 in the cold loop for non-ACGT bytes), looks its match masks up in shared memory, does its shifts as
    multiply-adds (IMAD.HI for bit 63) and has no divergence slow paths around its shuffles."""
    if not shutil.which("cuobjdump"):
        pytest.skip("cuobjdump not available")
    from racon_gpu_b200 import api
    api.load_library()
    out = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True, check=True).stdout
    solo = _function_section(out, "aln_split_kernel")
    assert solo.count("SHFL.UP") >= 17
    assert "LDS.64" in solo and "IMAD.HI.U32" in solo
    assert solo.count("BRA.DIV") == 0 and solo.count("WARPSYNC.COLLECTIVE") == 0
    n_instr = len(re.findall(r"^\s+/\*[0-9a-f]{4,6}\*/", solo, flags=re.M))
    assert n_instr < 3600, f"aln_split_kernel grew to {n_instr} instructions"
    team = _function_section(out, "aln_split_team_kernel")
    assert "BAR.SYNC" in team or "BAR.SYNC.DEFER_BLOCKING" in team  # the teams' named barriers
