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

``args['segments']`` (``run_predict.py --segments``) also writes ``NISQA_segments.csv`` into ``output_dir``: one row per
segment of every file with its time span, its score under each pooling head and the head's pooling weight
(:meth:`nisqa_b200.scorer.Scorer.segments`).  Single process only.

``args['embeddings']`` (``run_predict.py --embeddings``) also writes ``NISQA_embeddings.npz`` into ``output_dir``: the
file column (``files``; NISQA_DE also ``references``), the head names (``heads``, the ``*_pred`` columns) and each file's
pooled vector under every head (``pooled`` float32 [files, heads, width], :meth:`nisqa_b200.scorer.Scorer.embed`).
Single process only.

``args['window_s']`` / ``args['window_hop_s']`` (``run_predict.py --window_s S --window_hop_s S``) score every file as a
timeline of overlapping windows instead (:meth:`nisqa_b200.scorer.Scorer.windows`): ``predict()`` returns, and writes
to ``output_dir/NISQA_windows.csv``, one row per window with its time span, segment count and scores.  Files longer than
``ms_max_segments`` are accepted in this mode.  Single process only.  A double-ended checkpoint (``predict_csv`` with
``csv_ref``) scores window pairs of each file and its reference, the reference windows widened by
``args['reference_margin_s']`` seconds on either side (default 0): each row also has the reference file and the
reference window's time span and segment count.

``args['alignment']`` (``run_predict.py --alignment``, NISQA_DE in ``predict_csv`` mode with ``csv_ref``) also writes
``NISQA_alignment.csv`` into ``output_dir``: one row per degraded segment (in windows mode: per segment of every window
pair's degraded window) with the file and reference columns, ``seg``, ``t_start``, ``ref_seg``, ``ref_t_start``,
``delay_s``, ``weight``, ``centroid_delay_s`` and ``peak`` (:meth:`nisqa_b200.scorer.Scorer.align`).  Single process
only.
"""
import datetime
import os
from glob import glob

import numpy as np
import pandas as pd

pd.options.mode.chained_assignment = None

import torch

from . import NISQA_lib as NL
from . import evaluate as EV
from . import dist as nb_dist
from .engine import engine_from_checkpoint, load_checkpoint


class nisqaModel(object):
    """Loads the checkpoint into the engine and the table of files to predict."""

    def __init__(self, args):
        self.args = args
        if args.get("segments") and nb_dist.env_world()[1] > 1:
            raise ValueError("segments: NISQA_segments.csv is written by a single process, not under torchrun with %d ranks"
                             % nb_dist.env_world()[1])
        win = args.get("window_s") is not None or args.get("window_hop_s") is not None
        if win and nb_dist.env_world()[1] > 1:
            raise ValueError("window_s: NISQA_windows.csv is written by a single process, not under torchrun with %d ranks"
                             % nb_dist.env_world()[1])
        if win and (args.get("window_s") is None or args.get("window_hop_s") is None):
            raise ValueError("window_s / window_hop_s: windows need both, got window_s=%r, window_hop_s=%r"
                             % (args.get("window_s"), args.get("window_hop_s")))
        if args.get("embeddings") and nb_dist.env_world()[1] > 1:
            raise ValueError("embeddings: NISQA_embeddings.npz is written by a single process, not under torchrun with %d "
                             "ranks" % nb_dist.env_world()[1])
        if win and args.get("segments"):
            raise ValueError("segments: per-segment rows are not written in windows mode (window_s)")
        if win and args.get("embeddings"):
            raise ValueError("embeddings: pooled vectors are not written in windows mode (window_s)")
        if args.get("alignment") and nb_dist.env_world()[1] > 1:
            raise ValueError("alignment: NISQA_alignment.csv is written by a single process, not under torchrun with %d "
                             "ranks" % nb_dist.env_world()[1])
        if args.get("reference_margin_s") is not None and not win:
            raise ValueError("reference_margin_s: a margin of the reference windows needs windows mode (window_s)")
        if "mode" not in self.args:
            self.args["mode"] = "main"
        self.runinfos = {}
        self._getDevice()
        self._loadModel()
        if self.args.get("reference_margin_s") is not None and not self.args["double_ended"]:
            raise ValueError("reference_margin_s: a single-ended checkpoint reads no reference (NISQA_DE only)")
        if self.args.get("alignment") and not self.args["double_ended"]:
            raise ValueError("alignment: a single-ended checkpoint aligns no reference (NISQA_DE only)")
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
        if self.args.get("window_s") is not None:
            df = self.predict_windows()
            if self.args["output_dir"]:
                df.to_csv(os.path.join(self.args["output_dir"], "NISQA_windows.csv"), index=False)
                if self.args.get("alignment"):
                    self.predict_alignment().to_csv(os.path.join(self.args["output_dir"], "NISQA_alignment.csv"), index=False)
            print(df.to_string(index=False))
            return df
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
        if self.args.get("segments") and self.args["output_dir"]:
            self.predict_segments().to_csv(os.path.join(self.args["output_dir"], "NISQA_segments.csv"), index=False)
        if self.args.get("embeddings") and self.args["output_dir"]:
            np.savez(os.path.join(self.args["output_dir"], "NISQA_embeddings.npz"), **self.predict_embeddings())
        if self.args.get("alignment") and self.args["output_dir"]:
            self.predict_alignment().to_csv(os.path.join(self.args["output_dir"], "NISQA_alignment.csv"), index=False)
        return self.ds_val.df

    def predict_alignment(self):
        """-> DataFrame of ``NISQA_alignment.csv``: one row per degraded segment of every file pair, in file order (in
        windows mode: per segment of every window pair's degraded window, with the pair's ``window`` index and its
        ``win_t_start`` / ``win_ref_t_start`` after the file columns), from :meth:`Scorer.align`.  Pairs are batched and
        decoded as :meth:`predict_segments` (windows mode: one file pair per call, as :meth:`predict_windows`)."""
        sc = self._scorer()
        ds = self.ds_val
        col, col_ref = ds.filename_column, ds.filename_column_ref
        files, refs = ds.df[col].tolist(), ds.df[col_ref].tolist()
        win = self.args.get("window_s") is not None
        parts = {}

        def part(i, res, r0, n, extra):
            d = pd.DataFrame({col: [files[i]] * n, col_ref: [refs[i]] * n})
            for k, v in extra.items():
                d[k] = v
            d["seg"] = np.arange(n) if not win else np.concatenate([np.arange(c) for c in res.counts]) if n else []
            sl = slice(r0, r0 + n)
            d["t_start"], d["ref_seg"] = res.t_start[sl], res.ref_seg[sl].cpu().numpy()
            d["ref_t_start"], d["delay_s"] = res.ref_t_start[sl], res.delay_s[sl]
            d["weight"] = res.weight[sl].cpu().numpy().astype(float)
            d["centroid_delay_s"] = res.centroid_delay_s[sl]
            d["peak"] = res.peak[sl].cpu().numpy().astype(float)
            return d
        if win:
            for i in range(len(ds)):
                y, sr = NL.read_wav(ds.file_path(i), ds.ms_channel)
                y_ref, sr_ref = NL.read_wav(ds.file_path_ref(i), None)
                res = sc.align(self._batch_tensor([y])[0], sr, self._batch_tensor([y_ref])[0], reference_sample_rate=sr_ref,
                               window_s=self.args["window_s"], window_hop_s=self.args["window_hop_s"],
                               reference_margin_s=self.args.get("reference_margin_s") or 0.0)
                n = int(sum(res.counts))
                parts[i] = part(i, res, 0, n, {"window": res.window, "win_t_start": res.pair_t_start[res.window],
                                               "win_ref_t_start": res.pair_ref_t_start[res.window]})
        else:
            for batch, call in self._file_batches():
                res = call(sc.align)
                r0 = 0
                for j, i in enumerate(batch):
                    parts[i] = part(i, res, r0, res.counts[j], {})
                    r0 += res.counts[j]
        return pd.concat([parts[i] for i in range(len(ds))], ignore_index=True)

    def predict_segments(self):
        """-> DataFrame with one row per segment of every file, in file order: the file column, ``segment``,
        ``t_start`` / ``t_end`` (seconds), each head's segment score (``*_pred``) and pooling weight (``*_weight``).
        The files are decoded by the dataset's loader and scored in batches of ``tr_bs_val`` clips of one sample rate
        through :meth:`Scorer.segments`."""
        sc = self._scorer()
        ds = self.ds_val
        col = ds.filename_column
        files = ds.df[col].tolist()
        weight_cols = [c[:-len("_pred")] + "_weight" for c in sc.columns]
        parts = {}
        for batch, call in self._file_batches():
            res = call(sc.segments)
            s, w = res.seg_scores.cpu().numpy(), res.seg_weights.cpu().numpy()
            r0 = 0
            for j, i in enumerate(batch):
                n = res.counts[j]
                part = pd.DataFrame({col: [files[i]] * n, "segment": np.arange(n),
                                     "t_start": res.t_start[r0:r0 + n], "t_end": res.t_end[r0:r0 + n]})
                for h, c in enumerate(sc.columns):
                    part[c] = s[r0:r0 + n, h].astype(float)
                for h, c in enumerate(weight_cols):
                    part[c] = w[r0:r0 + n, h].astype(float)
                parts[i] = part
                r0 += n
        return pd.concat([parts[i] for i in range(len(ds))], ignore_index=True)

    def predict_embeddings(self):
        """-> dict of the arrays of ``NISQA_embeddings.npz``: ``files`` (the file column; NISQA_DE also ``references``,
        the reference column), ``heads`` (the ``*_pred`` names) and ``pooled`` float32 [files, heads, width], each
        file's pooled vector under every head (:meth:`Scorer.embed`), batched and decoded as :meth:`predict_segments`."""
        sc = self._scorer()
        ds = self.ds_val
        pooled = np.empty((len(ds), len(sc.columns), self.model.embedding_width()), dtype=np.float32)
        for batch, call in self._file_batches():
            pooled[batch] = call(sc.embed).pooled.cpu().numpy()
        out = {"files": np.array(ds.df[ds.filename_column].tolist()), "heads": np.array(sc.columns), "pooled": pooled}
        if ds.double_ended:
            out["references"] = np.array(ds.df[ds.filename_column_ref].tolist())
        return out

    def _scorer(self):
        """a Scorer over the loaded engine"""
        from .scorer import Scorer
        sc = Scorer.__new__(Scorer)
        sc._configure(self.args, self.dev)
        sc.engine = self.model
        return sc

    def _file_batches(self):
        """The files decoded by the dataset's loader, in batches of ``tr_bs_val`` clips of one sample rate (NISQA_DE: one
        pair of rates) -> (file indices, call), call(f) = f(wave, sr, lengths=..., reference...) on the batch"""
        ds, bs = self.ds_val, max(1, int(self.args["tr_bs_val"]))
        de = ds.double_ended
        loaded = []
        for i in range(len(ds)):
            y, sr = NL.read_wav(ds.file_path(i), ds.ms_channel)
            ref = NL.read_wav(ds.file_path_ref(i), None) if de else (None, None)
            loaded.append((y, sr) + ref)
        groups = {}
        for i, (_, sr, _, sr_ref) in enumerate(loaded):
            groups.setdefault((sr, sr_ref), []).append(i)
        for (sr, sr_ref), rows in groups.items():
            for k in range(0, len(rows), bs):
                batch = rows[k:k + bs]
                wave, lens = self._batch_tensor([loaded[i][0] for i in batch])
                kw = {}
                if de:
                    kw["reference"], kw["reference_lengths"] = self._batch_tensor([loaded[i][2] for i in batch])
                    kw["reference_sample_rate"] = sr_ref
                yield batch, lambda f, wave=wave, sr=sr, lens=lens, kw=kw: f(wave, sr, lengths=lens, **kw)

    def predict_windows(self):
        """-> DataFrame with one row per window of every file, in file order: the file column, ``t_start`` / ``t_end``
        (seconds), ``n_segments`` and each head's score (``*_pred``).  Each file is decoded by the dataset's loader and
        scored on its own through :meth:`Scorer.windows`.  NISQA_DE: one row per window pair, with the reference column
        after the file column and ``ref_t_start`` / ``ref_t_end`` / ``ref_n_segments`` of the reference window; the
        reference is read as the loader's mono mix."""
        sc = self._scorer()
        ds = self.ds_val
        col = ds.filename_column
        files = ds.df[col].tolist()
        de = ds.double_ended
        parts = []
        for i in range(len(ds)):
            y, sr = NL.read_wav(ds.file_path(i), ds.ms_channel)
            wave, _ = self._batch_tensor([y])
            kw = {}
            if de:
                y_ref, sr_ref = NL.read_wav(ds.file_path_ref(i), None)
                kw = {"reference": self._batch_tensor([y_ref])[0], "reference_sample_rate": sr_ref,
                      "reference_margin_s": self.args.get("reference_margin_s") or 0.0}
            res = sc.windows(wave, sr, self.args["window_s"], self.args["window_hop_s"], **kw)
            s = res.scores.cpu().numpy()
            part = pd.DataFrame({col: [files[i]] * res.counts[0]})
            if de:
                part[ds.filename_column_ref] = ds.df[ds.filename_column_ref].iloc[i]
            part["t_start"], part["t_end"] = res.t_start, res.t_end
            if de:
                part["ref_t_start"], part["ref_t_end"] = res.ref_t_start, res.ref_t_end
            part["n_segments"] = res.n_segments
            if de:
                part["ref_n_segments"] = res.ref_n_segments
            for h, c in enumerate(sc.columns):
                part[c] = s[:, h].astype(float)
            parts.append(part)
        return pd.concat(parts, ignore_index=True)

    def _batch_tensor(self, clips):
        """host clips -> ([B, T] CUDA tensor, lengths): int16 when every clip is int16, else float32"""
        if any(c.dtype != np.int16 for c in clips):
            clips = [c if c.dtype == np.float32 else c.astype(np.float32) / np.float32(32768.0) for c in clips]
        lens = [c.shape[0] for c in clips]
        x = np.zeros((len(clips), max(lens)), dtype=clips[0].dtype)
        for j, c in enumerate(clips):
            x[j, :lens[j]] = c
        return torch.from_numpy(x).to(self.dev), lens

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
        # checkpoint hyper-parameters, overridden by the caller's dict (model:941-942)
        self.args, state_dict = load_checkpoint(model_path, self.args)

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
        self.model = engine_from_checkpoint(self.args, state_dict, device=self.dev.index if self.dev.index is not None else 0)
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
