"""Plug allrank_b200 into an unmodified allRank checkout.

allRank resolves its hot-path callables by NAME at run time:
    loss   : getattr(allrank.models.losses, config.loss.name)        allrank/main.py:83
    metric : getattr(allrank.models.metrics, name)                   allrank/training/train_utils.py:50
    model  : allrank.models.model.make_model(...)                    allrank/main.py:75
so `patch_allrank()` only has to rebind those attributes; `allrank/main.py` and `train_utils.fit` then run
unchanged on the CUDA kernels.  (allRank must be importable; nothing here imports it otherwise.)

The callers either side of the path (SURVEY.md 8(f) ranks 3-4) are rebound the same way:
    epoch metrics : allrank.training.train_utils.{metric_on_epoch, compute_metrics}    train_utils.py:37-56
    rank_slates   : allrank.inference.inference_utils.rank_slates                      inference_utils.py:12-30
    slate loading : allrank.data.dataset_loading.{load_libsvm_dataset, create_data_loaders} (+ the names main.py
                    imported from it, main.py:8) -- opt-in (`patch_data=True`): the corpus then lives in HBM.
    click metrics : allrank.inference.inference_utils.metrics_on_clicked_slates                inference_utils.py:63-82
    clicks        : allrank.click_models.click_utils.click_on_slates -- opt-in (`patch_clicks=True`): random
                    click models then draw from a counter hash instead of numpy's stream.
    LibSVM saving : allrank.data.dataset_saving.write_to_libsvm_without_masked -- opt-in (`patch_write=True`): the
                    click-through files are formatted on the device, byte for byte what sklearn writes.
allrank/rank_and_click.py imports make_model, CustomDataParallel, rank_slates, metrics_on_clicked_slates,
click_on_slates and write_to_libsvm_without_masked by name (rank_and_click.py:11-18); those bindings are rebound too.
"""
import functools

from . import click_models as _click_models
from . import data as _data
from . import inference as _inference
from . import losses as _losses
from . import metrics as _metrics
from . import model as _model
from . import training as _training
from . import writer as _writer

LOSS_NAMES = ("listNet", "listMLE", "approxNDCGLoss", "lambdaLoss", "neuralNDCG", "neuralNDCG_transposed", "rankNet",
              "rankNet_weightByGTDiff", "rankNet_weightByGTDiff_pow", "binary_listNet", "pointwise_rmse", "bce",
              "ordinal", "with_ordinals")
METRIC_NAMES = ("ndcg", "dcg", "mrr")


_MODULES = {"losses": "allrank.models.losses", "metrics": "allrank.models.metrics", "model": "allrank.models.model",
            "main": "allrank.main", "train_utils": "allrank.training.train_utils",
            "inference_utils": "allrank.inference.inference_utils", "dataset_loading": "allrank.data.dataset_loading",
            "rank_and_click": "allrank.rank_and_click", "click_utils": "allrank.click_models.click_utils",
            "dataset_saving": "allrank.data.dataset_saving"}


def single_process_model(model):
    """Stands in for allrank.models.model_utils.CustomDataParallel when allrank/main.py:76-78 runs on a box with
    several visible GPUs.  The CUDA path scales as ONE PROCESS PER GPU (torchrun + allrank_b200.ddp.FlatDDP, a single
    NCCL all-reduce of the flat gradient); single-process nn.DataParallel would replicate a model whose parameters
    are views of one flat device buffer, which cannot work.  The model is returned unwrapped and trains on the device
    allRank selects (cuda:0 of the visible devices): launch one process per GPU with CUDA_VISIBLE_DEVICES / torchrun."""
    return model


def _rebind(saved, mod_key, name, fn):
    import importlib
    target = importlib.import_module(_MODULES[mod_key])
    saved[mod_key + "." + name] = getattr(target, name)
    setattr(target, name, fn)


def _import_rank_and_click():
    try:
        import allrank.rank_and_click  # noqa: F401
        return True
    except Exception:
        return False


def patch_allrank(patch_model=True, patch_eval=True, patch_data=False, patch_clicks=False, data_parser="sklearn",
                  patch_write=False):
    """Rebind allrank.models.{losses,metrics}.<name> (and make_model, the epoch-metric helpers, rank_slates,
    metrics_on_clicked_slates and -- opt-in -- the slate loaders, click_on_slates and write_to_libsvm_without_masked)
    to the CUDA implementations.
    data_parser: how the patched loaders read LibSVM files -- "sklearn" (the reference's parser on the host) or
    "device" (the CUDA parser of allrank_b200.data, same arrays bit for bit).
    Returns the dict of original callables so the caller can restore them."""
    if data_parser not in _data.PARSERS:
        raise ValueError("data_parser must be one of {}, got {!r}".format(_data.PARSERS, data_parser))
    import allrank.models.losses as ref_losses
    import allrank.models.metrics as ref_metrics
    import allrank.models.model as ref_model
    saved = {}
    for name in LOSS_NAMES:
        saved["losses." + name] = getattr(ref_losses, name)
        setattr(ref_losses, name, getattr(_losses, name))
    for name in METRIC_NAMES:
        saved["metrics." + name] = getattr(ref_metrics, name)
        setattr(ref_metrics, name, getattr(_metrics, name))
    if patch_model:
        saved["model.make_model"] = ref_model.make_model
        ref_model.make_model = _model.make_model
        try:                                   # allrank/main.py does `from allrank.models.model import make_model`
            import allrank.main as ref_main
            saved["main.make_model"] = ref_main.make_model
            ref_main.make_model = _model.make_model
            # main.py:76-78 wraps the model in CustomDataParallel when device_count() > 1: neutralised (see above)
            saved["main.CustomDataParallel"] = ref_main.CustomDataParallel
            ref_main.CustomDataParallel = single_process_model
        except Exception:
            pass
    have_rac = _import_rank_and_click()
    if patch_model and have_rac:           # rank_and_click.py:73,78-79: the same make_model / DataParallel bindings
        _rebind(saved, "rank_and_click", "make_model", _model.make_model)
        _rebind(saved, "rank_and_click", "CustomDataParallel", single_process_model)
    if patch_eval:
        _rebind(saved, "train_utils", "metric_on_epoch", _training.metric_on_epoch)
        _rebind(saved, "train_utils", "compute_metrics", _training.compute_metrics)
        _rebind(saved, "inference_utils", "rank_slates", _inference.rank_slates)
        # inference_utils bound the metrics at import (`from allrank.models.metrics import ndcg, dcg`); its
        # metrics_on_clicked_slates would call the CUDA metrics with host tensors
        _rebind(saved, "inference_utils", "metrics_on_clicked_slates", _inference.metrics_on_clicked_slates)
        if have_rac:
            _rebind(saved, "rank_and_click", "rank_slates", _inference.rank_slates)
            _rebind(saved, "rank_and_click", "metrics_on_clicked_slates", _inference.metrics_on_clicked_slates)
    if patch_clicks:
        _rebind(saved, "click_utils", "click_on_slates", _click_models.click_on_slates)
        if have_rac:
            _rebind(saved, "rank_and_click", "click_on_slates", _click_models.click_on_slates)
    if patch_write:
        _rebind(saved, "dataset_saving", "write_to_libsvm_without_masked", _writer.write_to_libsvm_without_masked)
        if have_rac:
            _rebind(saved, "rank_and_click", "write_to_libsvm_without_masked", _writer.write_to_libsvm_without_masked)
    if patch_data:
        loaders = {name: getattr(_data, name) for name in ("load_libsvm_dataset", "load_libsvm_dataset_role",
                                                           "load_libsvm_role", "create_data_loaders")}
        if data_parser != "sklearn":
            for name in ("load_libsvm_dataset", "load_libsvm_dataset_role", "load_libsvm_role"):
                loaders[name] = functools.partial(loaders[name], parser=data_parser)
        for name, fn in loaders.items():
            _rebind(saved, "dataset_loading", name, fn)
        try:
            _rebind(saved, "main", "load_libsvm_dataset", loaders["load_libsvm_dataset"])
            _rebind(saved, "main", "create_data_loaders", _data.create_data_loaders)
        except Exception:
            pass
    return saved


def unpatch_allrank(saved):
    import importlib
    for key, fn in saved.items():
        mod, name = key.split(".")
        setattr(importlib.import_module(_MODULES[mod]), name, fn)
