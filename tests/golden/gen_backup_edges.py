"""Generate tests/golden/backup_edges_golden.npz: the reference's own agents/cppmodule/core.cpp (compiled unchanged -> oracle/_ref/core*.so,
oracle/Makefile) backing up the designed trees of tests/backup_edges.py: traces of 1-512 levels around the engine's 32-level windows,
observations repeated on the trace and among the leaf's children, evaluator outputs and visit counts at their edges, four gammas, the
LP backup in both of the reference's forms and the single / vanilla backups.  The golden keeps what the backup changed and a digest
of each case's inputs; the tests regenerate the inputs with backup_edges.design().
Run:  python tests/golden/gen_backup_edges.py      (needs `make -C oracle ref`; a regeneration is byte-identical)"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")]
import oracle_py as O  # noqa: E402
import backup_edges as BE  # noqa: E402

OUT = os.path.join(HERE, "backup_edges_golden.npz")


def main():
    core = O.load_ref_module("core")
    cases = BE.design()
    outs = [BE.run(c, core) for c in cases]
    BE.save(OUT, cases, outs)
    print("backup_edges_golden: %d cases" % len(cases))


if __name__ == "__main__":
    main()
