# -*- coding: utf-8 -*-
"""Command line of the H100 NISQA engine.

Flag-compatible with the reference CLI (reference run_predict.py:8-43): the three predict modes
and the same option names, so existing invocations keep working:

    python run_predict.py --mode predict_file --pretrained_model weights/nisqa.tar --deg a.wav
    python run_predict.py --mode predict_dir  --pretrained_model weights/nisqa.tar --data_dir d --bs 64
    torchrun --nproc-per-node 8 run_predict.py --mode predict_csv ...   (one rank per GPU)
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
    args = vars(parser.parse_args(argv))

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
