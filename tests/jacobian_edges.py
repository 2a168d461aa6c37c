"""One table of the Jacobian kernels' shapes at the edges of their plans (TEST INFRASTRUCTURE ONLY), with a Python
mirror of their shared-memory layouts.

The three Jacobian kernels each size their own layout (csrc/qp_jac.cu jac_dims and box_jac_dims, csrc/qp_boxq.cu
boxq_jac_dims): a factor of S, M or the bordered K, and then as many warps' column buffers as the shared memory left
takes, `nblk` (at most the 8 warps of a CTA). A warp sweeps 8-column blocks t = warp, warp + nblk, ...; which blocks
exist and where they land in J depend on the rows / cols masks. The C ABI reports only the shared memory, so
jac_layout, box_layout and boxq_layout mirror the layouts, and tests/test_jacobian_edges_cpu.py checks that the mirror
gives the C functions' bytes over a grid and on every entry.

Entries, as the kernels plan them (smem in bytes; blocks: column blocks for the full masks; next: one step past the
edge, which the kernel does not cover or for which there is no plan; sweep: the entry runs the mask sweep of
tests/jacobian_edges_jobs.py):
- JAC (k_jacobian, the default plan_for plan): the nz = nineq edge, the widest S with a narrow nz, many equality tiles,
  the widest nz any plan takes (three column blocks in flight without equality rows), and three small shapes with all
  8 warps holding buffers: fewer blocks than warps, a partial last equality tile, h tiles starting at neq_pad = 8.
- BOX (k_box_jacobian): its own coverage limits, which are not the box forward's (2880 variables with one bound, 2616
  with both, nz = neq = 200; with e = 0 shared memory is filled to within 256..448 bytes of the cap), each reached by a
  forward on a cluster plan (`fwd` "cl4") or a distributed-M one ("dm2", "dm4": neq_pad > 128), and three one-CTA
  shapes ("one").
- BOXQ (k_boxq_jacobian): entries of tests/boxq_families.py. Its buffers are N x 8 beside a factor of order
  N = nz_pad + neq_pad <= 256, so it never runs with fewer than two warps: largest_lb is the fewest.
"""
import ctypes

JAC_MAX_SMEM = 232448 - 1024     # kJacMaxSmem (qp_jac.cu)
BOX_MAX_SMEM = 232448            # kBoxMaxSmem (qp_box_loop.cuh), k_boxq_jacobian's cap
WARPS = 256 // 32                # 256 threads per CTA in all three kernels
PAN_LD = 12                      # kPanLd (qp_pf.cuh)


def r8(v):
    return (v + 7) & ~7


def pf_elems(nts):
    return (32 * nts + 64) * nts


def pf_tab_doubles(nts):
    return (nts * (nts + 1) // 2 + 3) >> 2


def _buffers(head, per, cap):
    """warps holding a column buffer of `per` doubles once `head` doubles are taken, of `cap` bytes (at most 8)"""
    left = cap - 8 * head
    return min(left // (8 * per), WARPS) if left > 0 else 0


def jac_layout(n, m, e, ep, ms, msp):
    """jac_dims of a qpb200_plan's fields: (nblk, smem bytes, column blocks of the full masks)."""
    nts, np_ = msp >> 3, r8(n)
    blk = pf_elems(nts) + (8 * nts + 8) * PAN_LD + r8(pf_tab_doubles(nts)) + 8 * nts
    per = 8 * (np_ + msp)
    nb = _buffers(blk, per, JAC_MAX_SMEM) if m >= 1 else 0
    return nb, (8 * (blk + nb * per) if nb else 0), np_ // 8 + nts


def box_layout(n, e, has_lb, has_ub):
    """box_jac_dims: (nblk, smem bytes, column blocks of the full masks)."""
    m, nts, np_ = (int(has_lb) + int(has_ub)) * n, r8(e) >> 3, r8(n)
    blk = pf_elems(nts) + (8 * nts + 8) * PAN_LD + r8(pf_tab_doubles(nts)) + 8 * nts + np_ + r8(m)
    per = 8 * (np_ + 8 * nts)
    nb = _buffers(blk, per, JAC_MAX_SMEM)
    return nb, (8 * (blk + nb * per) if nb else 0), np_ // 8 + nts


def boxq_layout(n, e, has_lb, has_ub):
    """boxq_jac_dims: (nblk, smem bytes, column blocks of the full masks). A is staged in the buffers' space."""
    m, np_, ep = (int(has_lb) + int(has_ub)) * n, r8(n), r8(e)
    N = np_ + ep
    nts = N >> 3
    blk = r8(pf_elems(nts)) + r8((8 * nts + 8) * PAN_LD) + r8(pf_tab_doubles(nts)) + N + r8(m)
    per, a_end = 8 * N, blk + r8(e * (n | 1))
    nb = _buffers(blk, per, BOX_MAX_SMEM)
    if N > 256 or 8 * a_end > BOX_MAX_SMEM:
        nb = 0
    return nb, (8 * max(blk + nb * per, a_end) if nb else 0), np_ // 8 + ep // 8


def jac_plan_layout(plan):
    return jac_layout(plan.nz, plan.nineq, plan.neq, plan.neq_pad, plan.ms, plan.ms_pad)


# ---- the C functions ------------------------------------------------------------------------------------------------

def jac_plan(n, m, e):
    """(rc, plan) of qpb200_plan_init, uncached"""
    from qpth_b200 import _lib
    p = _lib.Plan()
    return _lib.load().qpb200_plan_init(n, m, e, ctypes.byref(p)), p


def jac_smem(plan):
    from qpth_b200 import _lib
    out = ctypes.c_int64(-1)
    assert _lib.load().qpb200_jacobian_smem(ctypes.byref(plan), ctypes.byref(out)) == 0
    return out.value


def box_plan(n, e, sides):
    """(rc, plan) of qpb200_box_plan_init, uncached (no cluster knob)"""
    from qpth_b200 import _lib
    p = _lib.BoxPlan()
    return _lib.load().qpb200_box_plan_init(n, e, int(sides != "ub"), int(sides != "lb"), ctypes.byref(p)), p


def box_smem(plan):
    from qpth_b200 import _lib
    out = ctypes.c_int64(-1)
    assert _lib.load().qpb200_box_jacobian_smem(ctypes.byref(plan), ctypes.byref(out)) == 0
    return out.value


def boxq_smem(plan):
    from qpth_b200 import _lib
    out = ctypes.c_int64(-1)
    assert _lib.load().qpb200_boxq_jacobian_smem(ctypes.byref(plan), ctypes.byref(out)) == 0
    return out.value


def box_forward(plan):
    """the forward layout of a box plan: "one", "cl<C>" (M replicated) or "dm<C>" (M distributed, neq_pad > 128)"""
    if plan.ok:
        return "one"
    if plan.cl_ctas:
        return ("dm%d" if plan.neq_pad > 128 else "cl%d") % plan.cl_ctas
    return "dense"


# ---- the table ------------------------------------------------------------------------------------------------------

def _j(shape, smem, nblk, blocks, nxt=None, sweep=False):
    return dict(shape=shape, smem=smem, nblk=nblk, blocks=blocks, next=nxt, sweep=sweep)


# k_jacobian, (nz, nineq, neq)
JAC = {
    "nz_eq_nineq": _j((200, 200, 0), 220672, 1, 50, (201, 201, 0), sweep=True),
    "narrow_widest_S": _j((8, 208, 0), 223296, 1, 27, (8, 209, 0)),
    "eq_one_tile": _j((192, 192, 8), 220160, 1, 49, (193, 193, 8)),
    "eq_five_tiles": _j((320, 160, 40), 228352, 1, 65, (322, 161, 40)),
    "eq_23_tiles": _j((248, 16, 184), 223744, 1, 56, (249, 16, 185), sweep=True),
    "widest_nz_eq": _j((1056, 8, 132), 185088, 1, 150, (1057, 8, 132)),
    "widest_nz": _j((1056, 1, 0), 206720, 3, 133, (1057, 1, 0), sweep=True),
    "small_few_blocks": _j((17, 13, 3), 31744, 8, 6, sweep=True),
    "small_partial_eq": _j((29, 8, 17), 43072, 8, 8, sweep=True),
    "small_h_after_pad": _j((45, 61, 3), 95168, 8, 15, sweep=True),
}

# k_box_jacobian, (nz, neq, sides)
BOX = {
    "widest_lb": dict(_j((2880, 0, "lb"), 231168, 1, 360, (2881, 0, "lb")), fwd="cl4"),
    "widest_ub": dict(_j((2880, 0, "ub"), 231168, 1, 360, (2881, 0, "ub")), fwd="cl4"),
    "widest_both": dict(_j((2616, 0, "both"), 230976, 1, 327, (2617, 0, "both")), fwd="cl4"),
    "most_eq_lb": dict(_j((200, 200, "lb"), 223872, 1, 50, (201, 201, "lb"), sweep=True), fwd="dm2"),
    "most_eq_ub": dict(_j((200, 200, "ub"), 223872, 1, 50, (201, 201, "ub")), fwd="dm2"),
    "most_eq_both": dict(_j((200, 200, "both"), 225472, 1, 50, (201, 201, "both")), fwd="dm2"),
    "dm_300_192": dict(_j((300, 192, "both"), 220096, 1, 62), fwd="dm2"),
    "dm_1000_160": dict(_j((1000, 160, "both"), 228736, 1, 145), fwd="dm4"),
    "one_31_13": dict(_j((31, 13, "both"), 29888, 8, 6, sweep=True), fwd="one"),
    "one_5_1": dict(_j((5, 1, "both"), 10816, 8, 2, sweep=True), fwd="one"),
    "one_64_40_lb": dict(_j((64, 40, "lb"), 68224, 8, 13, sweep=True), fwd="one"),
}

# k_boxq_jacobian: entries of tests/boxq_families.py (the shape and plan are theirs)
BOXQ = {
    "full_both": _j((144, 32, "both"), 224640, 6, 22, sweep=True),
    "full_odd_lb": _j((97, 71, "lb"), 223168, 6, 22),
    "tile_9": _j((64, 9, "both"), 81920, 8, 10, sweep=True),
    "tiny_1_1": _j((1, 1, "lb"), 12800, 8, 2, sweep=True),
    "largest_lb": _j((192, 1, "lb"), 222208, 2, 25, sweep=True),
}


def sides_flags(sides):
    return sides != "ub", sides != "lb"


def order(kind, shape):
    """n + 2m + e: the order of the dense model's system"""
    if kind == "jac":
        n, m, e = shape
    else:
        n, e, sides = shape
        m = n * (1 + (sides == "both"))
    return n + 2 * m + e
