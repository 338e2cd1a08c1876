import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100; run with -m gpu)")


@pytest.fixture(scope="session")
def oracle_engine():
    """Snapshot -> AllocateResult through the CPU oracle (test infrastructure)."""
    from oracle.pyoracle import OracleSession
    from volcano_b200.uthelper import AllocateResult

    def run(snap, threads=1):
        import numpy as np
        from oracle import pyoracle
        s = OracleSession(snap, threads=threads)
        actions = [a for a in snap.actions if a != "enqueue"]
        if "allocate" in actions or not any(a in ("preempt", "reclaim") for a in actions):
            dec, vis, fe = s.allocate()
        else:  # an action list without allocate (the reference's preempt / reclaim unit tests)
            dec, vis, fe = np.zeros(0, pyoracle.DECISION_DTYPE), np.zeros(0, pyoracle.VISIT_DTYPE), np.zeros(0, np.int32)
        res = AllocateResult(dec, vis, fe)
        for a in actions:  # the configured order (scheduler.go:124-153)
            if a == "backfill" and snap.B > 0:
                res.backfill = AllocateResult(*s.backfill())
            elif a == "preempt":
                res.preempt = AllocateResult(*s.preempt())
            elif a == "reclaim":
                res.reclaim = AllocateResult(*s.reclaim())
        if snap.hn_job_soft is not None and snap.hn_job_soft.any():
            import numpy as np
            from oracle import pyoracle
            res.job_allocated_hypernodes = np.array([pyoracle.lib().vco_job_allocated_hypernode(s.h, j) for j in range(snap.J)],
                                                    np.int32)
        s.close()
        return res

    return run
