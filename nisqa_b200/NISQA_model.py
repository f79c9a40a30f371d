"""``nisqaModel`` for the engine - the predict side of the reference driver class
(reference nisqa/NISQA_model.py:21-81, 732-847, 928-1051) with the same constructor argument
dict, the same ``predict()`` surface (prints, ``NISQA_results.csv``, returned DataFrame) and the
same precedence of checkpoint args vs. CLI args, but with the torch modules replaced by
:class:`nisqa_b200.engine.Engine`.

``evaluate()`` (reference model:48-52, 572-715) prints the reference's per-database statistics of the last
``predict()`` from :mod:`nisqa_b200.evaluate` (SURVEY.md 8f.3).  Out of scope here (SURVEY.md section 2):
``train()`` and ``mode == 'main'`` raise ``NotImplementedError``.  Double-ended checkpoints (NISQA_DE) run in
``predict_csv`` mode with ``args['csv_ref']`` naming the reference column, as in the reference (model:846, 951-955).  There is no CPU device: ``tr_device='cpu'``
or a machine without CUDA raises.
"""
import datetime
import os
from glob import glob

import pandas as pd

pd.options.mode.chained_assignment = None

import torch

from . import NISQA_lib as NL
from . import evaluate as EV
from . import dist as nb_dist
from .engine import Engine, config_from_args


class nisqaModel(object):
    """Loads the checkpoint into the engine and the table of files to predict."""

    def __init__(self, args):
        self.args = args
        if "mode" not in self.args:
            self.args["mode"] = "main"
        self.runinfos = {}
        self._getDevice()
        self._loadModel()
        self._loadDatasets()
        self.args["now"] = datetime.datetime.today()

    # ------------------------------------------------------------------ out of scope
    def train(self):
        raise NotImplementedError("training is outside the predict path (SURVEY.md section 2, #15)")

    # ------------------------------------------------------------------ evaluate (model:48-52, 572-715)
    def evaluate(self, mapping="first_order", do_print=True, do_plot=False):
        """Statistics of the predictions against the labels in the csv tables.  For dimension models one
        block per predicted dimension (db_results_val_<dim>, keys of ``self.r`` suffixed like the
        reference), for MOS-only models ``self.db_results`` / ``self.r``."""
        if nb_dist.env_world()[0] != 0:
            return
        con = self.ds_val.df_con is not None

        def block(title, target):
            print("--> %s:" % title)
            db_results, r = EV.eval_results(
                self.ds_val.df, dcon=self.ds_val.df_con, target_mos=target, target_ci=target + "_ci",
                pred=target + "_pred", mapping=mapping, do_print=do_print, do_plot=do_plot)
            if not con:
                print("r_p_mean_file: {:0.2f}, rmse_mean_file: {:0.2f}".format(r["r_p_mean_file"], r["rmse_mean_file"]))
            elif target == "noi":          # the reference prints two of the three numbers for this block (model:636)
                print("r_p_mean_con: {:0.2f}, rmse_mean_con: {:0.2f}".format(r["r_p_mean_con"], r["rmse_mean_con"]))
            else:
                print("r_p_mean_con: {:0.2f}, rmse_mean_con: {:0.2f}, rmse_star_map_mean_con: {:0.2f}".format(
                    r["r_p_mean_con"], r["rmse_mean_con"], r["rmse_star_map_mean_con"]))
            return db_results, r

        if self.args["dim"] != True:  # noqa: E712
            self.db_results, self.r = block("MOS", "mos")
            return
        self.r = {}
        for target in ("mos", "noi", "dis", "col", "loud"):
            db_results, r = block(target.upper(), target)
            setattr(self, "db_results_val_" + target, db_results)
            self.r.update(r if target == "mos" else {k + "_" + target: v for k, v in r.items()})
        r_mean = 1 / 5 * sum(self.r["r_p_mean_con" + sfx] for sfx in ("", "_noi", "_col", "_dis", "_loud"))
        print("\nAverage over MOS and dimensions: r_p={:0.3f}".format(r_mean))

    # ------------------------------------------------------------------ predict (model:54-81)
    def predict(self):
        rank, world, _ = nb_dist.env_world()
        chatty = rank == 0
        if chatty:
            print("---> Predicting ...")
        if self.args["dim"] == True:  # noqa: E712  (mirrors the reference comparison)
            y_val_hat, y_val = NL.predict_dim(
                self.model, self.ds_val, self.args["tr_bs_val"], self.dev,
                num_workers=self.args["tr_num_workers"])
        else:
            y_val_hat, y_val = NL.predict_mos(
                self.model, self.ds_val, self.args["tr_bs_val"], self.dev,
                num_workers=self.args["tr_num_workers"])

        if self.args["output_dir"]:
            self.ds_val.df["model"] = self.args["name"]
            if chatty:
                self.ds_val.df.to_csv(
                    os.path.join(self.args["output_dir"], "NISQA_results.csv"), index=False)
        if chatty:
            print(self.ds_val.df.to_string(index=False))
        return self.ds_val.df

    # ------------------------------------------------------------------ datasets (model:732-847)
    def _loadDatasets(self):
        mode = self.args["mode"]
        if mode == "predict_file":
            self._loadDatasetsFile()
        elif mode == "predict_dir":
            self._loadDatasetsFolder()
        elif mode == "predict_csv":
            self._loadDatasetsCSVpredict()
        elif mode == "main":
            raise NotImplementedError("mode 'main' (training CSVs) is outside the predict path")
        else:
            raise NotImplementedError("mode not available")

    def _dataset(self, df, data_dir, filename_column, df_con=None, filename_column_ref=None):
        a = self.args
        return NL.SpeechQualityDataset(
            df, df_con=df_con, data_dir=data_dir, filename_column=filename_column,
            mos_column="predict_only", seg_length=a["ms_seg_length"], max_length=a["ms_max_segments"],
            to_memory=None, to_memory_workers=None, seg_hop_length=a["ms_seg_hop_length"],
            transform=None, ms_n_fft=a["ms_n_fft"], ms_hop_length=a["ms_hop_length"],
            ms_win_length=a["ms_win_length"], ms_n_mels=a["ms_n_mels"], ms_sr=a["ms_sr"],
            ms_fmax=a["ms_fmax"], ms_channel=a["ms_channel"], double_ended=a["double_ended"],
            dim=a["dim"], filename_column_ref=filename_column_ref)

    def _loadDatasetsFolder(self):
        # unsorted glob of lower-case *.wav, basenames in column 'deg' (model:746-748)
        files = [os.path.basename(f) for f in glob(os.path.join(self.args["data_dir"], "*.wav"))]
        df_val = pd.DataFrame(files, columns=["deg"])
        if nb_dist.env_world()[0] == 0:
            print("# files: {}".format(len(df_val)))
        if len(df_val) == 0:
            raise ValueError("No wav files found in data_dir")
        if nb_dist.env_world()[1] > 1:
            # glob order is arbitrary; ranks must agree on the row order before sharding
            df_val = df_val.sort_values("deg").reset_index(drop=True)
        self.ds_val = self._dataset(df_val, self.args["data_dir"], "deg")

    def _loadDatasetsFile(self):
        data_dir = os.path.dirname(self.args["deg"])
        file_name = os.path.basename(self.args["deg"])
        df_val = pd.DataFrame([file_name], columns=["deg"])
        self.ds_val = self._dataset(df_val, data_dir, "deg")

    def _loadDatasetsCSVpredict(self):
        csv_file_path = os.path.join(self.args["data_dir"], self.args["csv_file"])
        dfile = pd.read_csv(csv_file_path)
        if "csv_con" in self.args and self.args["csv_con"] is not None:
            dcon = pd.read_csv(os.path.join(self.args["data_dir"], self.args["csv_con"]))
        else:
            dcon = None
        # double-ended checkpoints read the reference signal's column from args['csv_ref'] (model:846)
        self.ds_val = self._dataset(dfile, self.args["data_dir"], self.args["csv_deg"], df_con=dcon,
                                    filename_column_ref=self.args["csv_ref"])

    # ------------------------------------------------------------------ model (model:928-1030)
    def _loadModel(self):
        if not self.args.get("pretrained_model"):
            raise NotImplementedError("the engine only runs pretrained checkpoints")
        if os.path.isabs(self.args["pretrained_model"]):
            model_path = os.path.join(self.args["pretrained_model"])
        else:
            model_path = os.path.join(os.getcwd(), self.args["pretrained_model"])
        checkpoint = torch.load(model_path, map_location="cpu", weights_only=False)
        # checkpoint hyper-parameters, overridden by the caller's dict (model:941-942)
        checkpoint["args"].update(self.args)
        self.args = checkpoint["args"]

        if self.args["model"] == "NISQA_DIM":
            self.args["dim"] = True
            self.args["csv_mos_train"] = None
            self.args["csv_mos_val"] = None
        else:
            self.args["dim"] = False
        if self.args["model"] == "NISQA_DE":      # model:951-955
            self.args["double_ended"] = True
        else:
            self.args["double_ended"] = False
            self.args["csv_ref"] = None
        for k, v in (("output_dir", None), ("ms_channel", None), ("tr_bs_val", 1), ("tr_num_workers", 0)):
            self.args.setdefault(k, v)

        chatty = nb_dist.env_world()[0] == 0
        if chatty:
            print("Model architecture: " + self.args["model"])
        cfg = config_from_args(self.args, max_chunk_segments=self.args.get("b200_max_chunk_segments", 0))
        self.model = Engine(cfg, device=self.dev.index if self.dev.index is not None else 0)
        self.model.load_state_dict(checkpoint["model_state_dict"])   # strict: the engine names what is missing
        if chatty:
            print("Loaded pretrained model from " + self.args["pretrained_model"])

    # ------------------------------------------------------------------ device (model:1032-1051)
    def _getDevice(self):
        if self.args.get("tr_device") == "cpu":
            raise RuntimeError("the engine has no CPU path (tr_device='cpu' requested)")
        if not torch.cuda.is_available():
            raise RuntimeError("no CUDA device available: the engine has no CPU fallback")
        _, world, local = nb_dist.env_world()
        idx = local if world > 1 else torch.cuda.current_device()
        torch.cuda.set_device(idx)
        self.dev = torch.device("cuda", idx)
        if nb_dist.env_world()[0] == 0:
            print("Device: {}".format(torch.device("cuda")))
