"""Generate tests/golden/eval_golden.json from the UNMODIFIED reference statistics functions
(``nisqa.NISQA_lib.eval_results`` and helpers, reference lib:1469-1852); runs only in the build container.

    python -m oracle.make_eval_golden            # needs the reference checkout ($NISQA_REFERENCE_DIR, read-only)

Inputs: a seeded synthetic listening-test table (3 databases with 4-6 conditions, per-file and
per-condition MOS / dimension labels with confidence intervals, predictions = labels + noise + a
database-specific bias), one database without labels.  The per-file and per-condition tables are stored
in the golden file next to the reference's outputs, so the test needs neither the seed logic nor the
reference.  The reference was written for an older pandas: ``groupby('con').mean()`` on frames with
string columns raises in pandas >= 2, so the frames handed to it here hold numeric columns plus ``db``
only where the reference touches it (the condition mean of ``db`` is never used).
"""
import io
import json
import os
import sys

import numpy as np
import pandas as pd

from oracle.build_ref import reference_dir

REF = reference_dir()     # the reference checkout ($NISQA_REFERENCE_DIR); exits with a message when absent
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import librosa_compat  # noqa: E402

MAPPINGS = [None, "first_order", "second_order", "third_order_not_monotonic", "third_order"]
TARGETS = ["mos", "noi", "dis", "col", "loud"]
CASE_TARGETS = ["mos", "noi"]          # eval_results cases; the driver-level blocks below cover all five


def make_tables(seed=0):
    rng = np.random.default_rng(seed)
    files, cons = [], []
    for k, (db, n_con, per_con, labelled) in enumerate([("DB_A", 6, 8, True), ("DB_B", 4, 12, True), ("DB_C", 5, 6, True),
                                                       ("DB_unlab", 3, 4, False)]):
        for c in range(1, n_con + 1):
            q = rng.uniform(1.3, 4.7)
            rowsc = []
            for f in range(per_con):
                row = {"db": db, "con": c, "filepath_deg": "%s/c%02d_f%02d.wav" % (db, c, f)}
                for t in TARGETS:
                    lab = float(np.clip(q + rng.normal(0, 0.35), 1, 5))
                    row[t] = lab if labelled else np.nan
                    row[t + "_pred"] = float(np.clip(0.85 * lab + 0.4 + 0.1 * k + rng.normal(0, 0.3), 1, 5))
                rowsc.append(row)
            files.extend(rowsc)
            con = {"db": db, "con": c}
            for t in TARGETS:
                vals = np.array([r[t] for r in rowsc])
                con[t] = float(vals.mean()) if labelled else np.nan
                con[t + "_ci"] = float(0.3 * 1.96 * vals.std(ddof=1) / np.sqrt(per_con)) if labelled else np.nan
            cons.append(con)
    return pd.DataFrame(files), pd.DataFrame(cons)


class _NumericGroupFrame(pd.DataFrame):
    """The reference calls ``df_db.groupby('con').mean()`` on the per-file table (pandas < 2 dropped
    non-numeric columns silently); hand it a view whose groupby only sees numeric columns."""
    @property
    def _constructor(self):
        return _NumericGroupFrame

    def groupby(self, *a, **k):
        num = pd.DataFrame(self).select_dtypes("number")
        return num.groupby(*a, **k)


def main():
    librosa_compat.install()
    sys.path.insert(0, REF)
    import nisqa.NISQA_lib as NL
    dfile, dcon = make_tables()
    cases = []
    for target in CASE_TARGETS:
        for mapping in MAPPINGS:
            for with_con in (True, False):
                df = _NumericGroupFrame(dfile.copy())
                buf = io.StringIO()
                old = sys.stdout
                sys.stdout = buf
                try:
                    db_res, overall = NL.eval_results(df, dcon=dcon.copy() if with_con else None, target_mos=target,
                                                      target_ci=target + "_ci", pred=target + "_pred", mapping=mapping,
                                                      do_print=True, do_plot=False)
                finally:
                    sys.stdout = old
                cases.append({"target": target, "mapping": mapping, "with_con": with_con,
                              "db_results": json.loads(db_res.to_json(orient="split")),
                              "overall": {k: (None if np.isnan(v) else float(v)) for k, v in overall.items()},
                              "y_hat_map": [None if np.isnan(v) else float(v) for v in df["y_hat_map"].to_numpy()],
                              "printed": buf.getvalue()})
    # driver level: the reference's nisqaModel.evaluate() on a stub instance (no checkpoint, no audio)
    from nisqa.NISQA_model import nisqaModel

    class _DS(object):
        pass
    driver = []
    for dim in (True, False):
        for with_con in (True, False):
            m = object.__new__(nisqaModel)
            m.args = {"dim": dim}
            m.ds_val = _DS()
            m.ds_val.df = _NumericGroupFrame(dfile.copy())
            m.ds_val.df_con = dcon.copy() if with_con else None
            buf = io.StringIO()
            old = sys.stdout
            sys.stdout = buf
            try:
                m.evaluate(mapping="first_order", do_print=True, do_plot=False)
            finally:
                sys.stdout = old
            driver.append({"dim": dim, "with_con": with_con, "printed": buf.getvalue(),
                           "r": {k: (None if np.isnan(v) else float(v)) for k, v in m.r.items()}})
    # helper-level vectors
    rng = np.random.default_rng(3)
    y = rng.uniform(1, 5, 40); yh = np.clip(y + rng.normal(0, 0.4, 40), 1, 5); ci = rng.uniform(0.05, 0.4, 40)
    helpers = {"y": y.tolist(), "y_hat": yh.tolist(), "ci": ci.tolist(),
               "rmse_d0": float(NL.calc_rmse(y, yh)), "rmse_d3": float(NL.calc_rmse(y, yh, d=3)),
               "rmse_star_d1": float(NL.calc_rmse_star(y, yh, ci, 1)[0]),
               "b1": NL.fit_first_order(y, yh).tolist(), "b2": NL.fit_second_order(y, yh).tolist(),
               "b3": NL.fit_third_order(y, yh).tolist(),
               "mapped_b3": NL.calc_mapped(yh, NL.fit_third_order(y, yh)).tolist(),
               "is_const": [bool(NL.is_const(np.ones(5) * 2.5)), bool(NL.is_const(y))]}
    out = {"dfile": json.loads(dfile.to_json(orient="split")), "dcon": json.loads(dcon.to_json(orient="split")),
           "cases": cases, "driver": driver, "helpers": helpers}
    dst = os.path.join(ROOT, "tests", "golden", "eval_golden.json")
    json.dump(out, open(dst, "w"))
    print("wrote", dst, os.path.getsize(dst), "bytes,", len(cases), "cases")


if __name__ == "__main__":
    main()
