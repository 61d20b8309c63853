"""graphlearn_b200.engine - see the package README / DESIGN.md for the layer map.

The fused CUDA trainers are importable from here: ``FastSageTrainer`` (supervised node classification) and
``FastLinkSageTrainer`` (unsupervised link prediction)."""

__all__ = ["FastSageTrainer", "FastLinkSageTrainer"]


def __getattr__(name):
    # resolved on first use, so that importing a sibling module does not pull in every trainer
    if name == "FastSageTrainer":
        from .fast_sage import FastSageTrainer
        return FastSageTrainer
    if name == "FastLinkSageTrainer":
        from .fast_link_sage import FastLinkSageTrainer
        return FastLinkSageTrainer
    raise AttributeError("module %r has no attribute %r" % (__name__, name))
