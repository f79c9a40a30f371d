# -*- coding: utf-8 -*-
"""Scores a labelled corpus with the engine and prints the reference's evaluation statistics
(reference run_evaluate.py: predict_csv, then per-database Pearson / RMSE / mapped RMSE / RMSE*).

    python run_evaluate.py --pretrained_model weights/nisqa.tar --data_dir corpus --csv_file NISQA_corpus_file.csv \
        --csv_con NISQA_corpus_con.csv --csv_deg filepath_deg [--mapping first_order] [--bs 40] [--num_workers 6]

The per-file table needs the label columns (``mos`` and, for dimension models, ``noi dis col loud``) and a
``db`` column; with ``--csv_con`` both tables also need ``con`` (the condition number), and the
per-condition table the ``*_ci`` confidence-interval columns used by RMSE*.
"""
import argparse

from nisqa_b200.NISQA_model import nisqaModel


def parse_args(argv=None):
    ap = argparse.ArgumentParser(description="NISQA evaluation on H100")
    ap.add_argument("--pretrained_model", required=True)
    ap.add_argument("--data_dir", required=True)
    ap.add_argument("--csv_file", required=True, help="per-file table (paths + labels)")
    ap.add_argument("--csv_con", default=None, help="per-condition table (optional)")
    ap.add_argument("--csv_deg", required=True, help="column of the per-file table holding the wav paths")
    ap.add_argument("--csv_mos_val", default="mos")
    ap.add_argument("--output_dir", default=None)
    ap.add_argument("--bs", type=int, default=40)
    ap.add_argument("--num_workers", type=int, default=6)
    ap.add_argument("--ms_channel", type=int, default=None)
    ap.add_argument("--mapping", default="first_order",
                    choices=["none", "first_order", "second_order", "third_order_not_monotonic", "third_order"])
    ap.add_argument("--plot", action="store_true", help="scatter plots per database (needs matplotlib)")
    a = vars(ap.parse_args(argv))
    a["mode"] = "predict_csv"
    a["tr_bs_val"], a["tr_num_workers"] = a.pop("bs"), a.pop("num_workers")
    return a


if __name__ == "__main__":
    args = parse_args()
    mapping = args.pop("mapping")
    mapping = None if mapping == "none" else mapping
    plot = args.pop("plot")
    nisqa = nisqaModel(args)
    nisqa.predict()
    nisqa.evaluate(mapping=mapping, do_print=True, do_plot=plot)
