# -*- coding: utf-8 -*-
"""Command line of the H100 NISQA engine.

Flag-compatible with the reference CLI (reference run_predict.py:8-43): the three predict modes
and the same option names, so existing invocations keep working:

    python run_predict.py --mode predict_file --pretrained_model weights/nisqa.tar --deg a.wav
    python run_predict.py --mode predict_dir  --pretrained_model weights/nisqa.tar --data_dir d --bs 64
    torchrun --nproc-per-node 8 run_predict.py --mode predict_csv ...   (one rank per GPU)
    python run_predict.py --mode predict_dir ... --output_dir out --segments   (+ out/NISQA_segments.csv)
    python run_predict.py --mode predict_dir ... --output_dir out --embeddings   (+ out/NISQA_embeddings.npz)
    python run_predict.py --mode predict_dir ... --output_dir out --window_s 10 --window_hop_s 1   (out/NISQA_windows.csv)
    python run_predict.py --mode predict_csv --pretrained_model de.tar --csv_file t.csv --csv_deg deg --csv_ref ref \
        --output_dir out --window_s 10 --window_hop_s 1 --reference_margin_s 0.5   (NISQA_DE window pairs)
    python run_predict.py --mode predict_csv --pretrained_model de.tar --csv_file t.csv --csv_deg deg --csv_ref ref \
        --output_dir out --alignment   (+ out/NISQA_alignment.csv: each degraded segment's reference segment and delay)
"""
import argparse

from nisqa_b200.NISQA_model import nisqaModel

# option name -> (type, default, what it is)
_OPTIONS = {
    "mode": (str, None, "predict_file | predict_dir | predict_csv"),
    "pretrained_model": (str, None, "checkpoint (.tar) to load; relative paths resolve against the working directory"),
    "deg": (str, None, "wav file to score (predict_file)"),
    "data_dir": (str, None, "directory holding the wav files (predict_dir) / base directory of the csv paths"),
    "output_dir": (str, None, "if given, NISQA_results.csv is written here"),
    "csv_file": (str, None, "table of files to score (predict_csv)"),
    "csv_deg": (str, None, "name of the csv column with the file paths"),
    "csv_ref": (str, None, "NISQA_DE: name of the csv column with the reference file paths (default: the checkpoint's)"),
    "num_workers": (int, 0, "native wav-decode threads per batch"),
    "bs": (int, 1, "clips per engine call"),
    "ms_channel": (int, None, "channel to use for multi-channel files (default: mono mix)"),
}
_REQUIRED = {"mode", "pretrained_model"}
# what each mode cannot run without; the messages are the reference's own (reference run_predict.py:22-37) so that
# scripts matching on them keep working
_NEEDS = {
    "predict_file": [("deg", "--deg argument with path to input file needed")],
    "predict_dir": [("data_dir", "--data_dir argument with folder with input files needed")],
    "predict_csv": [("csv_file", "--csv_file argument with csv file name needed"),
                    ("csv_deg", "--csv_deg argument with csv column name of the filenames needed")],
}


def parse_args(argv=None):
    parser = argparse.ArgumentParser(description="NISQA speech quality prediction on H100")
    for name, (typ, default, text) in _OPTIONS.items():
        parser.add_argument("--" + name, type=typ, default=default, required=name in _REQUIRED, help=text)
    parser.add_argument("--segments", action="store_true",
                        help="also write NISQA_segments.csv into output_dir: every segment's time span, score and "
                             "pooling weight (single process only)")
    parser.add_argument("--embeddings", action="store_true",
                        help="also write NISQA_embeddings.npz into output_dir: each file's pooled vector under every "
                             "pooling head, the input of its last Linear (single process only)")
    parser.add_argument("--alignment", action="store_true",
                        help="NISQA_DE: also write NISQA_alignment.csv into output_dir: for every degraded segment (of "
                             "every window pair with --window_s) the reference segment it matched, the delay in seconds "
                             "and the match's weight and score (single process only)")
    parser.add_argument("--window_s", type=float, default=None,
                        help="score every file as a timeline of windows of this many seconds (with --window_hop_s) and "
                             "write NISQA_windows.csv into output_dir; files of any length (single process only)")
    parser.add_argument("--window_hop_s", type=float, default=None, help="hop between window starts in seconds")
    parser.add_argument("--reference_margin_s", type=float, default=None,
                        help="NISQA_DE windows: widen each reference window by this many seconds on either side, so "
                             "that delayed content near a window's edge is found (default 0)")
    args = vars(parser.parse_args(argv))
    if args["csv_ref"] is None:
        del args["csv_ref"]                       # (the checkpoint's column stays)
    if args["reference_margin_s"] is not None:
        if args["window_s"] is None:
            raise ValueError("--reference_margin_s argument needs --window_s and --window_hop_s")
        if not args["reference_margin_s"] >= 0:
            raise ValueError("--reference_margin_s argument must be a non-negative number of seconds, not %r"
                             % args["reference_margin_s"])
    else:
        del args["reference_margin_s"]
    if (args["window_s"] is None) != (args["window_hop_s"] is None):
        missing = "window_hop_s" if args["window_hop_s"] is None else "window_s"
        raise ValueError("--%s argument needed: --window_s and --window_hop_s go together" % missing)
    for key in ("window_s", "window_hop_s"):
        if args[key] is not None and not args[key] > 0:
            raise ValueError("--%s argument must be a positive number of seconds, not %r" % (key, args[key]))

    if args["mode"] not in _NEEDS:
        raise NotImplementedError("--mode given not available")
    for key, complaint in _NEEDS[args["mode"]]:
        if args[key] is None:
            raise ValueError(complaint)
    if args["mode"] == "predict_csv" and args["data_dir"] is None:
        args["data_dir"] = ""                     # csv paths are then taken as given
    # the driver class reads the batch size / worker count under their training-config names
    args["tr_bs_val"], args["tr_num_workers"] = args["bs"], args["num_workers"]
    return args


if __name__ == "__main__":
    import os
    from nisqa_b200 import dist as nb_dist
    # the CLI process only feeds the GPU: keep it (and its pinned batch buffers) on the GPU's NUMA node
    nb_dist.bind_to_gpu_numa(int(os.environ.get("LOCAL_RANK", "0")))
    nisqa = nisqaModel(parse_args())
    nisqa.predict()
    # orderly exit under torchrun: every rank is past the score gather before any communicator goes away (the engine's
    # NCCL communicator first, then torch.distributed's) - a rank that simply exits can leave its peers hanging in
    # communicator teardown
    nb_dist.shutdown(nisqa.model)
