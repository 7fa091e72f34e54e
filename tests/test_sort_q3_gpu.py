"""-m gpu checks of Q3Pipeline's opt-in ORDER BY revenue DESC, o_orderdate ASC (and ORDER BY ... LIMIT 10) on one rank:
the output is in the comparator's order (tests/sort_ref.py) and holds the same groups as the unordered run and as the
oracle."""
import pytest

from tests import q3_util
from tests import sort_ref as sr

pytestmark = pytest.mark.gpu

KEYS, DESC = [3, 1], [True, False]


def _run(gu, tables, **kw):
    from galaxysql_b200 import pipelines
    cust, orders, line = tables
    q3 = pipelines.Q3Pipeline(gu.ctx(), customer_capacity=8000, orders_capacity=60000, lineitem_capacity=220000, nslabs=3,
                              expected_groups=4096, **kw)
    gu.ctx().profile(True)
    gu.ctx().profile_reset()
    out = gu.to_numpy(q3.run(gu.to_device(cust), gu.to_device(orders), gu.to_device(line)))
    prof = gu.ctx().profile_dump()
    gu.ctx().profile(False)
    stats = q3.stats
    q3.close()
    return out, stats, prof, q3.Q3_OUT_TYPES


@pytest.mark.parametrize("limit", [None, 10])
def test_q3_ordered_matches_unordered_run_and_oracle(limit):
    from tests import gpu_util as gu
    tables = q3_util.q3_tables(0, 1, ncust=8000, nord=60000, nline=220000)
    plain, _, prof0, types = _run(gu, tables)
    assert "k_sort_gather" not in prof0  # the default path runs no sort
    out, stats, prof, _ = _run(gu, tables, order_by=True, limit=limit)
    assert "k_sort_gather" in prof and (limit is None or "k_topn_hist" in prof)
    sr.check_ordered(out, out, types, KEYS, DESC)
    exp = q3_util.q3_oracle(*tables)
    for ref in (plain, exp):
        ref = [(c[0], None) for c in ref]
        if limit is not None:
            p = sr.lexsort_perm(ref, types, KEYS, DESC)[:limit]
            ref = [(c[0][p], None) for c in ref]
        gu.approx_rows_equal(out, ref, float_cols=[3], key_cols=[0, 1, 2], rtol=1e-6)
    assert stats["ordered_rows"] == (stats["groups"] if limit is None else limit)
