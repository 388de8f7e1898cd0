"""diffusers' step-end callback classes (``diffusers.callbacks``), restated without importing diffusers, and how the
denoise loop runs them.

* ``PipelineCallback(cutoff_step_ratio=1.0, cutoff_step_index=None)``: the base class, with diffusers' argument
  checks and messages; ``config`` holds the two values.
* ``MultiPipelineCallbacks(callbacks)``: the callbacks in list order; ``tensor_inputs`` is the concatenation of theirs.
* ``SDXLCFGCutoffCallback``: stops classifier-free guidance after step ``cutoff_step_index``, else
  ``int(pipe.num_timesteps * cutoff_step_ratio)``.

``DiffSenseiPipeline`` does not call a CFG cutoff's ``callback_fn`` (it would slice the condition tensors, which the
captured graph holds): ``resolve`` turns the callback into entries, and the loop applies a cutoff itself — at step k
it sets ``pipe._guidance_scale = 0.0`` at the cutoff's place in the list, and steps k + 1 .. run the UNet on the text
rows only with a guidance-free step.  diffusers' own ``SDXLCFGCutoffCallback`` and ``MultiPipelineCallbacks``
instances are recognised by class name and module and read through ``config`` / ``callbacks``; any other class from
diffusers' callbacks module is refused.
"""
from __future__ import annotations

from typing import Any, Dict, List, NamedTuple, Optional

# the condition tensors a CFG cutoff slices in diffusers; the engine keeps every sample's positive rows itself
CFG_CUTOFF_INPUTS = ("prompt_embeds", "add_text_embeds", "add_time_ids")
_DIFFUSERS = "diffusers.callbacks"


class _Config(dict):
    """diffusers' ``FrozenDict`` config as far as callbacks use it: item and attribute access."""

    def __getattr__(self, name):
        try:
            return self[name]
        except KeyError as e:
            raise AttributeError(name) from e


class PipelineCallback:
    """diffusers' ``PipelineCallback``: exactly one of ``cutoff_step_ratio`` (a float in [0, 1]) and
    ``cutoff_step_index`` is given, so passing only an index needs ``cutoff_step_ratio=None``."""

    def __init__(self, cutoff_step_ratio=1.0, cutoff_step_index=None):
        if (cutoff_step_ratio is None and cutoff_step_index is None) or (
                cutoff_step_ratio is not None and cutoff_step_index is not None):
            raise ValueError("Either cutoff_step_ratio or cutoff_step_index should be provided, not both or none.")
        if cutoff_step_ratio is not None and (
                not isinstance(cutoff_step_ratio, float) or not (0.0 <= cutoff_step_ratio <= 1.0)):
            raise ValueError("cutoff_step_ratio must be a float between 0.0 and 1.0.")
        self.config = _Config(cutoff_step_ratio=cutoff_step_ratio, cutoff_step_index=cutoff_step_index)

    @property
    def tensor_inputs(self) -> List[str]:
        raise NotImplementedError(f"You need to set the attribute `tensor_inputs` for {self.__class__}")

    def callback_fn(self, pipeline, step_index, timestep, callback_kwargs) -> Dict[str, Any]:
        raise NotImplementedError(f"You need to implement the method `callback_fn` for {self.__class__}")

    def __call__(self, pipeline, step_index, timestep, callback_kwargs) -> Dict[str, Any]:
        return self.callback_fn(pipeline, step_index, timestep, callback_kwargs)


class MultiPipelineCallbacks:
    """diffusers' ``MultiPipelineCallbacks``: each callback gets the previous one's kwargs, in list order."""

    def __init__(self, callbacks: List[PipelineCallback]):
        self.callbacks = callbacks

    @property
    def tensor_inputs(self) -> List[str]:
        return [name for callback in self.callbacks for name in callback.tensor_inputs]

    def __call__(self, pipeline, step_index, timestep, callback_kwargs) -> Dict[str, Any]:
        for callback in self.callbacks:
            callback_kwargs = callback(pipeline, step_index, timestep, callback_kwargs)
        return callback_kwargs


def cutoff_step(config, num_timesteps: int) -> int:
    """The step after which a CFG cutoff turns guidance off: ``cutoff_step_index``, else
    ``int(num_timesteps * cutoff_step_ratio)`` (``num_timesteps``: the steps the denoise runs, after img2img's
    ``strength``)."""
    if config.cutoff_step_index is not None:
        return config.cutoff_step_index
    return int(num_timesteps * config.cutoff_step_ratio)


class SDXLCFGCutoffCallback(PipelineCallback):
    """diffusers' ``SDXLCFGCutoffCallback``.  ``callback_fn`` is diffusers' (it keeps the last row of each condition
    tensor, right for one sample); ``DiffSenseiPipeline`` applies the cutoff itself and keeps every sample's rows."""

    tensor_inputs = list(CFG_CUTOFF_INPUTS)

    def callback_fn(self, pipeline, step_index, timestep, callback_kwargs) -> Dict[str, Any]:
        if step_index == cutoff_step(self.config, pipeline.num_timesteps):
            for name in self.tensor_inputs:
                callback_kwargs[name] = callback_kwargs[name][-1:]
            pipeline._guidance_scale = 0.0
        return callback_kwargs


class CfgCutoff(NamedTuple):
    """A CFG cutoff as the denoise loop applies it: the callback's ``config``."""
    config: Any


def _diffusers_name(cb) -> Optional[str]:
    """The class name of an instance of a class defined in diffusers' callbacks module, else None."""
    t = type(cb)
    return t.__name__ if t.__module__ == _DIFFUSERS else None


def _is_pipeline_callback(cb) -> bool:
    return isinstance(cb, PipelineCallback) or any(
        c.__name__ == "PipelineCallback" and c.__module__ == _DIFFUSERS for c in type(cb).__mro__)


def _entries(cb) -> list:
    name = _diffusers_name(cb)
    if isinstance(cb, MultiPipelineCallbacks) or name == "MultiPipelineCallbacks":
        return [e for c in cb.callbacks for e in _entries(c)]
    if isinstance(cb, SDXLCFGCutoffCallback) or name == "SDXLCFGCutoffCallback":
        return [CfgCutoff(cb.config)]
    if name is not None:
        raise ValueError(f"`callback_on_step_end`: diffusers' {name} is not supported (supported: "
                         "SDXLCFGCutoffCallback, MultiPipelineCallbacks and callbacks that read only `latents`)")
    return [cb]


def resolve(callback, tensor_inputs):
    """(entries, tensor_inputs) of a ``callback_on_step_end``.  A plain function (or None): (None, the given
    ``tensor_inputs``).  A ``PipelineCallback`` or ``MultiPipelineCallbacks`` (ours or diffusers'): its callbacks in
    call order, each a ``CfgCutoff`` or a callable, and the tensor inputs of the callables — their own
    ``tensor_inputs`` replace the keyword, as in diffusers, and a cutoff's names are satisfied by the engine."""
    multi = isinstance(callback, MultiPipelineCallbacks) or _diffusers_name(callback) == "MultiPipelineCallbacks"
    if callback is None or not (multi or _is_pipeline_callback(callback) or _diffusers_name(callback)):
        return None, tensor_inputs
    entries = _entries(callback)
    inputs = [n for e in entries if not isinstance(e, CfgCutoff) for n in e.tensor_inputs]
    return entries, inputs
