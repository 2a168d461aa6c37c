"""Throughput-mode setup (k_setup_pf at 192 threads, three per SM): its shared memory fits the slot of the three-per-SM
forward / backward CTAs wherever the library dispatches it, and every other three-per-SM shape keeps a setup kernel of its
own. Plan arithmetic only (no GPU)."""
import pytest

SM_TOTAL = 233472           # 228 KB of shared memory per SM
CTA_MAX = 232448 - 1024     # 227 KB opt-in per CTA, minus the library's slack
STATIC_SMEM = 16            # k_setup_pf's static shared memory (the SPD flag), as ptxas reports it


@pytest.fixture(scope="module")
def lib():
    from qpth_b200 import build, _lib
    build.build()
    return _lib.load()


def _throughput_setup(p):
    """What qpb200_pre_factor_kkt dispatches to for a plan in throughput mode (mirrors pre_factor_impl)."""
    if p.tiny:
        return "tiny"
    if p.pf and p.pf_three and p.pf3_ok and p.setup_pf_smem_bytes <= p.pf3_smem_bytes:
        return "pf192"
    if p.pf and p.setup_pf:
        return "pf256"
    if p.setup_fast:
        return "fast"
    return "resident" if p.smem_resident else "global"


def test_c2_setup_fits_the_forward_slot(lib):
    from qpth_b200 import _lib
    p = _lib.plan_for(100, 100, 0, two=True)
    assert p.pf_three == 1
    assert p.setup_pf_smem_bytes == 60928 and _throughput_setup(p) == "pf192"
    assert 3 * (p.setup_pf_smem_bytes + STATIC_SMEM + 1024) <= SM_TOTAL
    assert _lib.plan_for(100, 100, 0).setup_pf == 0          # latency mode keeps k_setup_fast at C2
    assert _throughput_setup(_lib.plan_for(50, 50, 10, two=True)) == "pf192"          # C3


def test_three_per_sm_shapes_fit_or_fall_back(lib):
    from qpth_b200 import _lib
    seen = {"pf192": 0, "other": 0}
    for nz in (8, 24, 40, 50, 64, 100, 104, 105, 112, 120, 136, 160, 200):
        for nineq in (8, 20, 50, 100, 150, 184):
            for neq in (0, 3, 10, 16):
                p = _lib.plan_for(nz, nineq, neq, two=True)
                if not (p.pf and p.pf3_ok):
                    continue
                tag = (nz, nineq, neq)
                got = _throughput_setup(p)
                if got == "pf192":
                    assert p.setup_pf_smem_bytes <= p.pf3_smem_bytes, tag
                    assert 3 * (p.setup_pf_smem_bytes + STATIC_SMEM + 1024) <= SM_TOTAL, tag
                    seen["pf192"] += 1
                else:                                        # the plan's own setup kernel, which must fit a CTA
                    assert p.setup_pf_smem_bytes > p.pf3_smem_bytes, tag
                    if got == "pf256":
                        assert p.setup_pf_smem_bytes <= CTA_MAX, tag
                    elif got in ("fast", "resident"):
                        assert p.setup_smem_bytes <= CTA_MAX, tag
                    else:
                        assert got == "global" and p.setup_scratch_elems > 0, tag
                    seen["other"] += 1
    assert seen["pf192"] > 0 and seen["other"] > 0, seen      # the grid reaches both sides of the choice
