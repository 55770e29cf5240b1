"""Minimal stand-in for pytorch_lightning 1.5 (SURVEY.md 8f-1): what the reference's inference scripts touch —
`LightningModule` as an nn.Module with `save_hyperparameters` / `.hparams` / `.device`
(/root/reference/lidiff/tools/diff_completion_pipeline.py:7,15-19,69).  Training orchestration (`Trainer`, DDP,
checkpoint callbacks; train.py:88-121) is out of scope (DESIGN.md §6) and raises."""
from .core.lightning import LightningModule  # noqa: F401


class LightningDataModule:
    """A plain base class: the reference's data modules (lidiff/datasets/datasets_refine.py) subclass it and define their own
    prepare_data / setup / *_dataloader methods."""

    def __init__(self, *args, **kwargs):
        pass

    def prepare_data(self):
        pass

    def setup(self, stage=None):
        pass


class Trainer:
    def __init__(self, *a, **k):
        raise NotImplementedError("lidiff_b200 shims pytorch_lightning for inference only; training (SURVEY.md 8f-3) is not built")


__version__ = "1.5.10+lidiff_b200.shim"
