"""CPU: the kernel choice table of tests/kernel_choice_cases.py against the claim-unit planner (fbr_plan_query, host
only).  Every case must land in the cell it names -- the kernel of the restated selection rule and the edge of that
kernel's index arithmetic -- and every cell must be run at each task count it lists, so a change to the selection rule, to
the planner or to the table fails here instead of silently dropping a kernel or a branch from the GPU suite."""
import pytest

from fiber_b200 import _abi

from . import kernel_choice_cases as K


def test_case_ids_are_unique():
    assert len(K.BY_ID) == len(K.CASES)


@pytest.mark.parametrize("cid", sorted(K.BY_ID))
def test_case_lands_in_its_cell(cid):
    c = K.BY_ID[cid]
    pred, _ = K.CELLS[c.cell]
    plan = K.case_plan(c)
    kernel = K.kernel_of(c)
    assert pred(c, plan, kernel), "%s: kernel %s, unit %d, slot %d, %d units" % (cid, kernel, plan.unit_tasks, plan.slot_stride, plan.n_units)


def test_every_cell_is_run_at_every_task_count():
    seen = {cell: set() for cell in K.CELLS}
    for c in K.CASES:
        assert c.cell in K.CELLS, c.id
        seen[c.cell] |= K.kinds_of(c, K.case_plan(c))
    for cell, (_, kinds) in K.CELLS.items():
        assert kinds <= seen[cell], "%s misses %s" % (cell, sorted(kinds - seen[cell]))


def test_cells_cover_every_kernel_and_dispatch_path():
    kernels = {K.kernel_of(c) for c in K.CASES}
    assert kernels == {"direct", "flat", "rows", "bulk"}
    dispatch = {K.expected_dispatch(c.body, c.arg_stride) for c in K.CASES if c.body in K.PAYLOAD}
    assert dispatch == {"tma", "regs", "checksum"}
    strided = {(c.arg_stride, c.args, c.place) for c in K.CASES if c.cell == "payload/strided_map"}
    for stride in (4112, 8192, 12288):
        for args in ("host", "dev"):
            for place in ("direct", "ring", "shuffle"):
                assert (stride, args, place) in strided
    # group tails: at least one case of each group size whose last ticket group is partial
    for g in (3, 32):
        assert any(K.case_plan(c).n_units % g and K.case_plan(c).n_units > g for c in K.CASES if c.cell == "bulk/group_%d" % g)


def test_rule_restatement_edges():
    """expected_kernel at hand-made plans: the selection rule's own edges, independent of the planner."""
    P = _abi.Plan

    def plan(unit, slot):
        p = P()
        p.unit_tasks, p.slot_stride = unit, slot
        return p
    ring, res = _abi.FBR_VIA_RING, _abi.FBR_RESILIENT
    assert K.expected_kernel(plan(32, 32 * 4096), 4096, 0, 0) == "direct"
    assert K.expected_kernel(plan(32, 32 * 4096), 4096, ring, 0) == "bulk"
    assert K.expected_kernel(plan(32, 32 * 4096), 4096, res, 0) == "rows"
    assert K.expected_kernel(plan(32, 32 * 4096), 4096, _abi.FBR_OUT_DEVICE, 4) == "flat"
    assert K.expected_kernel(plan(32, 32 * 4096), 4096, _abi.FBR_OUT_DEVICE, 16) == "direct"
    assert K.expected_kernel(plan(1, 4096), 4096, ring, 0) == "rows"
    assert K.expected_kernel(plan(1, 16384), 16384, ring, 0) == "bulk"            # the smallest slot of the bulk kernel
    assert K.expected_kernel(plan(5, 20480), 4096, ring, 0) == "rows"             # > 16 KB, no multiple
    assert K.expected_kernel(plan(3, 16), 4, ring, 0) == "flat"                   # slot rounded up to 16 B
    assert K.expected_kernel(plan(3, 16), 4, 0, 0) == "flat"                      # 12 B units: no direct
    assert K.expected_kernel(plan(1, 16), 4, 0, 0) == "direct"
    assert K.expected_dispatch("payload_map_4k", 4096) == "tma"
    assert K.expected_dispatch("payload_map_4k", 4112) == "regs"
