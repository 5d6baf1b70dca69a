"""Run the reference's UNCHANGED ``src/main.py`` with the kernel-backed model classes substituted.

    python -m rechorus_b200.overlay --ref /path/to/ReChorus/src --model_name BPRMF --emb_size 64 --lr 1e-3 \
        --l2 1e-6 --dataset Grocery_and_Gourmet_Food --path /tmp/data/ [--table_mode fused]

What it does (SURVEY.md section 8b1): puts the reference ``src/`` on ``sys.path``, restores the NumPy aliases the
reference still uses (np.object / np.int / np.float), imports the reference's model modules, builds classes
that graft this package's kernel mixins onto the reference's own ``GeneralModel`` / ``SequentialModel`` (so the
reference's Dataset, reader, runner, argument plumbing and checkpoint code are the ones that run), replaces
``models.general.BPRMF.BPRMF`` etc. with them, and ``runpy``s ``main.py``.  With ``--fused_step 1``,
``--device_metrics 1``, ``--device_batches N`` or ``--device_rec 1`` on the command line it also registers ``helpers.B200Runner`` (a subclass of the reference's own
BaseRunner) through the same by-name discovery, and ``helpers.B200ImpressionRunner`` (a subclass of its ImpressionRunner)
for the impression models.  Needs a CUDA device for the first forward call; there is no CPU
fallback.  ``--ref`` defaults to the unmodified copy build() stages in oracle/_ref/src (oracle/stage_reference.py).
"""
from __future__ import annotations

import os
import runpy
import sys

_HERE = os.path.dirname(os.path.abspath(__file__))
DEFAULT_REF = os.path.join(os.path.dirname(_HERE), "oracle", "_ref", "src")       # oracle/stage_reference.py


def _make_runner_module(ref_runner_cls):
    """``helpers.B200Runner``: the reference's own BaseRunner (train / evaluate / predict / print_res / logging
    untouched) with two seams re-pointed at the kernels, selected by flags the unchanged ``main.py`` parses for us
    (``main.py:164-176`` resolves the runner by the model's ``runner`` attribute and lets it add arguments):
      --fused_step 1      fit() = one C call per batch (model.train_step: forward, loss, backward, row-sparse optimizer;
                          next batch's index plan prefetched) instead of the loop body of BaseRunner.py:185-207
                          (fit() takes the stand-alone runner's dispatch, runner._routed_fit);
      --device_metrics 1  evaluate() ranks on the GPU (model.eval_ranks) instead of shipping predictions to the host;
      --device_batches N  fit() = the epoch's negatives, row shuffle and collate (SASRec's histories included) as device
                          kernels, seed N (runner.BaseRunner.fit_on_device) on the reference's own Dataset and corpus;
      --device_rec 1      the final top-100 lists of save_rec_results (main.py:117-132, TopK mode) computed on the GPU
                          (runner.BaseRunner.recommend) and written by runner.BaseRunner.save_rec_results.
    Without those flags every method is the reference's."""
    import types

    from . import runner as ours

    class B200Runner(ref_runner_cls):
        @staticmethod
        def parse_runner_args(parser):
            parser = ref_runner_cls.parse_runner_args(parser)
            parser.add_argument("--fused_step", type=int, default=0,
                                help="1 (with --table_mode fused): one C call per training step (model.train_step)")
            parser.add_argument("--device_metrics", type=int, default=0,
                                help="1: rank the ground truth on the GPU (model.eval_ranks)")
            parser.add_argument("--device_batches", type=int, default=0,
                                help="non-zero (a value > 1 is the seed): negatives, row shuffle and collate of every "
                                     "training batch on the GPU (runner.fit_on_device)")
            parser.add_argument("--device_rec", type=int, default=0,
                                help="1: compute the final top-k recommendation lists of save_rec_results on the GPU "
                                     "(TopK mode; the CSV is written on the host, byte-identical in format)")
            return parser

        def __init__(self, args):
            super().__init__(args)
            self.fused_step = getattr(args, "fused_step", 0)
            self.device_metrics = getattr(args, "device_metrics", 0)
            self.device_batches = getattr(args, "device_batches", 0)
            self.device_rec = getattr(args, "device_rec", 0)
            if self.device_rec:
                _install_device_rec()

        def fit(self, dataset, epoch=-1):
            loss = ours._routed_fit(self, dataset, epoch)
            return super().fit(dataset, epoch) if loss is None else loss

        def evaluate(self, dataset, topks, metrics):
            if self.device_metrics and hasattr(dataset.model, "eval_ranks"):
                return ours.BaseRunner.evaluate_on_device(self, dataset, topks, metrics)
            return super().evaluate(dataset, topks, metrics)

        recommend = ours.BaseRunner.recommend
        save_rec_results = ours.BaseRunner.save_rec_results

    mod = types.ModuleType("helpers.B200Runner")
    mod.B200Runner = B200Runner
    return mod


def _make_impression_runner_module(ref_runner_cls):
    """``helpers.B200ImpressionRunner``: the reference's own ImpressionRunner (predict / print_res / logging untouched)
    with two seams re-pointed at the device by flags the unchanged ``main.py`` parses for us:
      --device_metrics 1  evaluate() collates the batches and computes NDCG / MAP / HR on the GPU
                          (runner.impression_device_route says when; runner.evaluate_impression_on_device does it);
      --device_batches N  fit() builds every training batch and its labels on the GPU in the reference DataLoader's own
                          order (runner.impression_train_device_route says when; runner.fit_impression_on_device does it).
    Every other call is the reference's."""
    import types

    from . import runner as ours

    class B200ImpressionRunner(ref_runner_cls):
        @staticmethod
        def parse_runner_args(parser):
            parser = ref_runner_cls.parse_runner_args(parser)
            parser.add_argument("--device_metrics", type=int, default=0,
                                help="1: collate the evaluation batches and compute NDCG / MAP / HR on the GPU")
            parser.add_argument("--device_batches", type=int, default=0,
                                help="non-zero: collate every training batch and its labels on the GPU, in the order the "
                                     "host route shuffles them; the value is not a seed here (nothing is sampled)")
            return parser

        def __init__(self, args):
            super().__init__(args)
            self.device_metrics = getattr(args, "device_metrics", 0)
            self.device_batches = getattr(args, "device_batches", 0)

        def fit(self, data, epoch=-1):
            if ours.impression_train_device_route(self, data):
                return ours.fit_impression_on_device(self, data, epoch)
            return super().fit(data, epoch)

        def evaluate(self, data, topks, metrics, check_sort_idx=0, all=0):
            if ours.impression_device_route(self, data, check_sort_idx, all):
                return ours.evaluate_impression_on_device(self, data, topks)
            return super().evaluate(data, topks, metrics, check_sort_idx, all)

    mod = types.ModuleType("helpers.B200ImpressionRunner")
    mod.B200ImpressionRunner = B200ImpressionRunner
    return mod


def _install_device_rec() -> None:
    """Point the running main.py's module-level save_rec_results at the device route.  While runpy executes main.py it
    is sys.modules["__main__"], and main() looks the function up in those globals at call time (main.py:91-93), so
    main.py itself stays unmodified.  Only the TopK mode (--model_mode '' or TopK) is replaced; the CTR and
    Impression branches, and models without the kernel mixins' ``recommend``, keep the reference's function."""
    import logging
    main_mod = sys.modules.get("__main__")
    init_args = getattr(main_mod, "init_args", None)
    ref_fn = getattr(main_mod, "save_rec_results", None)
    if init_args is None or ref_fn is None or getattr(init_args, "model_mode", None) not in ("", "TopK"):
        return

    def save_rec_results(dataset, runner_, topk):
        if not hasattr(dataset.model, "recommend"):                 # not a kernel-backed model: the reference's route
            return ref_fn(dataset, runner_, topk)
        # the result path of main.py:99-101
        model_name = "{0}{1}".format(init_args.model_name, init_args.model_mode)
        result_path = os.path.join(runner_.log_path, runner_.save_appendix, "rec-{}-{}.csv".format(model_name,
                                                                                              dataset.phase))
        logging.info("Saving top-{} recommendation results to: {}".format(topk, result_path))
        runner_.save_rec_results(dataset, result_path, topk, sep=main_mod.args.sep)

    main_mod.save_rec_results = save_rec_results


def install(ref_src: str = DEFAULT_REF, b200_runner: bool = False):
    import numpy as np
    for alias, typ in (("object", object), ("int", int), ("float", float)):
        if not hasattr(np, alias):
            setattr(np, alias, typ)          # removed in NumPy >= 1.24; BaseModel.py:141, SASRec.py:69, utils.py:65
    if ref_src not in sys.path:
        sys.path.insert(0, ref_src)
    import models.BaseModel as RB                       # the reference's own base classes
    import models.general.BPRMF as ref_bprmf
    import models.general.NeuMF as ref_neumf
    import models.sequential.SASRec as ref_sasrec
    from . import plugin

    class BPRMF(plugin.BPRMFKernels, RB.GeneralModel):
        reader, runner = "BaseReader", "BaseRunner"
        extra_log_args = ["emb_size", "batch_size"]

        @staticmethod
        def parse_model_args(parser):
            parser = plugin.BPRMFKernels.parse_model_args(parser)
            return RB.GeneralModel.parse_model_args(parser)

        def __init__(self, args, corpus):
            RB.GeneralModel.__init__(self, args, corpus)
            self._base_init(args, corpus)

    class NeuMF(plugin.NeuMFKernels, RB.GeneralModel):
        reader, runner = "BaseReader", "BaseRunner"
        extra_log_args = ["emb_size", "layers"]

        @staticmethod
        def parse_model_args(parser):
            parser = plugin.NeuMFKernels.parse_model_args(parser)
            return RB.GeneralModel.parse_model_args(parser)

        def __init__(self, args, corpus):
            RB.GeneralModel.__init__(self, args, corpus)
            self._neumf_init(args, corpus)

    class SASRec(plugin.SASRecKernels, RB.SequentialModel):
        reader, runner = "SeqReader", "BaseRunner"
        extra_log_args = ["emb_size", "num_layers", "num_heads"]

        @staticmethod
        def parse_model_args(parser):
            parser = plugin.SASRecKernels.parse_model_args(parser)
            return RB.SequentialModel.parse_model_args(parser)

        def __init__(self, args, corpus):
            RB.SequentialModel.__init__(self, args, corpus)
            self._base_init(args, corpus)

    ref_bprmf.BPRMF, ref_neumf.NeuMF, ref_sasrec.SASRec = BPRMF, NeuMF, SASRec
    # --model_mode Impression (main.py:164: '{0}.{0}{1}'): the reference's own ImpressionModel / ImpressionSeqModel hosts
    # (flags, reader, runner, Dataset) with the forward on the kernels and the list-wise loss as one kernel family
    import models.BaseImpressionModel as RI

    class _ImpLoss:
        def loss(self, out_dict, target=None):
            from . import ops
            # ImpressionRunner.fit builds its labels with .int() (ImpressionRunner.py:187-190); the kernel reads int64
            return ops.listwise_loss(out_dict["prediction"], target.long(), self.loss_n, self.train_max_pos_item)

    class BPRMFImpression(_ImpLoss, plugin.BPRMFKernels, RI.ImpressionModel):
        reader, runner = "ImpressionReader", "ImpressionRunner"
        extra_log_args = ["emb_size", "batch_size"]

        @staticmethod
        def parse_model_args(parser):
            parser = plugin.BPRMFKernels.parse_model_args(parser)
            return RI.ImpressionModel.parse_model_args(parser)

        def __init__(self, args, corpus):
            RI.ImpressionModel.__init__(self, args, corpus)
            self.__dict__["_b2r_vectors"] = True
            self._base_init(args, corpus)

    class SASRecImpression(_ImpLoss, plugin.SASRecKernels, RI.ImpressionSeqModel):
        reader, runner = "ImpressionSeqReader", "ImpressionRunner"
        extra_log_args = ["emb_size", "num_layers", "num_heads"]

        @staticmethod
        def parse_model_args(parser):
            parser = plugin.SASRecKernels.parse_model_args(parser)
            return RI.ImpressionSeqModel.parse_model_args(parser)

        def __init__(self, args, corpus):
            RI.ImpressionSeqModel.__init__(self, args, corpus)
            self.__dict__["_b2r_vectors"] = True
            self._base_init(args, corpus)

    ref_bprmf.BPRMFImpression, ref_sasrec.SASRecImpression = BPRMFImpression, SASRecImpression
    if b200_runner:
        # main.py:10 `from helpers import *` imports what helpers.__all__ names; add the runner module there and let
        # the model classes choose it (main.py:166: eval('{0}.{0}'.format(model_name.runner)))
        import helpers
        import helpers.BaseRunner as ref_runner
        import helpers.ImpressionRunner as ref_imp_runner
        for name, mod, classes in (("B200Runner", _make_runner_module(ref_runner.BaseRunner), (BPRMF, NeuMF, SASRec)),
                                   ("B200ImpressionRunner", _make_impression_runner_module(ref_imp_runner.ImpressionRunner),
                                    (BPRMFImpression, SASRecImpression))):
            sys.modules["helpers." + name] = mod
            setattr(helpers, name, mod)
            if name not in helpers.__all__:
                helpers.__all__.append(name)
            for cls in classes:
                cls.runner = name
    return {"BPRMF": BPRMF, "NeuMF": NeuMF, "SASRec": SASRec, "BPRMFImpression": BPRMFImpression,
            "SASRecImpression": SASRecImpression}


def main(argv=None):
    argv = list(sys.argv[1:] if argv is None else argv)
    ref = DEFAULT_REF
    if "--ref" in argv:
        i = argv.index("--ref")
        ref = argv[i + 1]
        del argv[i:i + 2]
    # the runner seams only matter when one of their flags is on the command line; otherwise the reference's own
    # BaseRunner class is the one main.py instantiates
    flags = ("--fused_step", "--device_metrics", "--device_batches", "--device_rec")
    want_runner = any(a in flags or a.startswith(tuple(f + "=" for f in flags)) for a in argv)
    install(ref, b200_runner=want_runner)
    sys.argv = [os.path.join(ref, "main.py")] + argv
    runpy.run_path(os.path.join(ref, "main.py"), run_name="__main__")


if __name__ == "__main__":
    main()
