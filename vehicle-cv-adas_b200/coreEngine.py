"""coreEngine.py -- engine abstraction with the reference's protocol, backed by libadas_b200.

Mirrors /root/reference coreEngine.py: `EngineBase` (7-39: path check, `framework_type` property, the three
abstract methods) and the concrete-engine surface of TensorRTEngine (120-157) / OnnxEngine (159-186):
`providers`, `engine_dtype`, `get_engine_input_shape()`, `get_engine_output_shape()`, `engine_inference(x)`.
`B200Engine` accepts a `.b200w` plan (written by `adas_b200.plan`) or the reference's own `.onnx` model file, which is
converted once to a cached plan by `adas_b200.onnx_import` (the counterpart of convertOnnxToTensorRT.py); `.trt` engines are
TensorRT-private binaries and are not readable.
"""
import abc
import os

import numpy as np

from . import _capi


class EngineBase(abc.ABC):
    """Supports .b200w plans and ONNX model files (the reference supports Onnx/TensorRT, coreEngine.py:12-14)."""

    SUFFIXES = (".b200w", ".onnx")

    def __init__(self, model_path):
        if not os.path.isfile(model_path):
            raise Exception("The model path [%s] can't not found!" % model_path)
        assert model_path.endswith(self.SUFFIXES), "Parameters must be a .b200w or .onnx file."
        self._framework_type = None

    @property
    def framework_type(self):
        if self._framework_type is None:
            raise Exception("Framework type can't be None")
        return self._framework_type

    @framework_type.setter
    def framework_type(self, value):
        if not isinstance(value, str):
            raise Exception("Framework type need be str")
        self._framework_type = value

    @abc.abstractmethod
    def get_engine_input_shape(self):
        return NotImplemented

    @abc.abstractmethod
    def get_engine_output_shape(self):
        return NotImplemented

    @abc.abstractmethod
    def engine_inference(self):
        return NotImplemented


class B200Engine(EngineBase):
    """Drop-in for TensorRTEngine / OnnxEngine: same methods, sm_90a kernels underneath.

    device    replaces the hard-coded cuda.Device(0) of coreEngine.py:47 (defaults to LOCAL_RANK or 0)
    max_batch the reference is batch-1; batched calls are an extension (per-frame results are identical)
    """

    OUTPUT_NAMES = {0: ["output0"], 1: ["output0"], 2: ["loc_row", "loc_col", "exist_row", "exist_col"], 4: ["output0"], 5: ["output0"]}

    def __init__(self, plan_path, device=None, max_batch=1, conv_impl=0):
        EngineBase.__init__(self, plan_path)
        if device is None:
            device = int(os.environ.get("LOCAL_RANK", "0"))
        if plan_path.endswith(".onnx"):
            from .onnx_import import plan_from_onnx
            plan_path = plan_from_onnx(plan_path)        # parsed and packed once, cached next to the temp dir (ADAS_B200_PLAN_CACHE)
        self.plan_path = plan_path
        self.handle = _capi.Engine(plan_path, device=device, max_batch=max_batch, conv_impl=conv_impl)
        self.providers = "B200ExecutionProvider(sm_90a)"
        self.framework_type = "b200"
        self.engine_dtype = np.float32          # the input binding is fp32 NCHW; arithmetic is fp16 x fp16 -> fp32
        self.device = device
        self.max_batch = max_batch
        self.__input_shape = list(self.handle.input_shape)
        self.__output_shapes = [list(s) for s in self.handle.output_shapes]
        self.__output_names = list(self.OUTPUT_NAMES[self.handle.model_kind])

    def get_engine_input_shape(self):
        return self.__input_shape

    def get_engine_output_shape(self):
        return self.__output_shapes, self.__output_names

    def engine_inference(self, input_tensor):
        x = np.asarray(input_tensor)
        if x.ndim == 3:
            x = x[None]
        return self.handle.infer(x.astype(np.float32, copy=False))
