"""The dense-Q box-QP plan at its edges without a GPU: every entry of tests/boxq_families.py reproduces its plan figures
(qpb200_boxq_plan_init), one step past each edge is not ok, and the table agrees with tests/test_boxq_cpu.LARGEST."""
import pytest

from tests.boxq_families import ENTRIES, MAX_ORDER, MAX_SMEM, check_entry, dense_entries, edges, next_shape, plan_init

# what each edge is the edge of: one more variable (the width edges), one more equality row (the neq edges) or both
# (the entries that leave no byte of shared memory)
EDGE_OF = {"widest_both": "nz", "widest_lb": "nz", "widest_ub": "nz", "largest_lb": "nz", "largest_ub": "nz",
           "largest_both": "nz", "full_both": "both", "full_odd_lb": "both", "full_ub": "both", "most_eq_lb": "neq",
           "most_eq_both": "neq"}


@pytest.mark.parametrize("name", list(ENTRIES))
def test_entry_plan(name):
    p = check_entry(name)
    nz, neq, sides = ENTRIES[name]["shape"]
    assert (p.nz, p.neq, p.nineq, p.threads) == (nz, neq, nz * (1 + (sides == "both")), MAX_ORDER)


def test_every_edge_says_what_it_is_the_edge_of():
    assert sorted(EDGE_OF) == sorted(edges())


@pytest.mark.parametrize("name", edges())
def test_one_step_past_each_edge(name):
    """One more variable past the width edges, one more equality row past the neq edges, either past the entries that
    leave no byte: not ok, because shared memory runs out (the order stays within the 256 rows of the sweeps). `past`
    lists exactly the steps that are not ok: the other one stays ok."""
    ent = ENTRIES[name]
    nz, neq, sides = ent["shape"]
    rc, p = plan_init(nz, neq, sides)
    assert rc == 0 and p.ok == 1
    of = EDGE_OF[name]
    assert ({"nz", "neq"} if of == "both" else {of}) <= set(ent["past"]), (name, ent["past"])
    if of == "both":
        assert p.smem_bytes == MAX_SMEM, name
    for dim in ("nz", "neq"):
        rc, q = plan_init(*next_shape(ent["shape"], dim))
        assert rc == 0
        if dim in ent["past"]:
            assert q.ok == 0 and q.order <= MAX_ORDER and q.smem_bytes > MAX_SMEM, (name, dim)
        else:
            assert q.ok == 1, (name, dim)


@pytest.mark.parametrize("name", dense_entries())
def test_dense_entries_are_one_step_past_an_edge(name):
    shape = ENTRIES[name]["shape"]
    rc, p = plan_init(*shape)
    assert rc == 0 and p.ok == 0 and p.order <= MAX_ORDER and p.smem_bytes > MAX_SMEM
    assert any(next_shape(ENTRIES[k]["shape"], "nz") == shape for k in edges()), name


def test_table_agrees_with_largest():
    from tests.test_boxq_cpu import LARGEST
    shapes = {ENTRIES[k]["shape"]: k for k in edges()}
    for shape in LARGEST:
        assert shape in shapes, shape
        assert EDGE_OF[shapes[shape]] == "nz" and "nz" in ENTRIES[shapes[shape]]["past"]


def test_every_shape_has_neq_at_most_nz():
    for name, ent in ENTRIES.items():
        nz, neq, _ = ent["shape"]
        assert neq <= nz, name
