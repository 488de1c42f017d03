"""The linear maps and the gated MLP the fsb200 models share: forward and hand-written backward over views into the flat
buffers (fsb200/flat.py); and the int8 / int4 projection of the inference-only models (load_in_8bit / load_in_4bit)."""
import torch

from .. import lib as L
from .. import ops


class Linear:
    """One linear map of a model: the weight (one parameter, or a fused span of adjacent ones such as q|k|v or w1|w3), its
    gradient view exactly as the flat buffers handed it out, and optionally a bias and its gradient view. ZeRO-2's compaction
    re-points those views in place, not tensors derived from them (`.view(-1)`, a slice), so none is kept here.
    An HF `Linear` weight is [out, in] (forward NT, dgrad NN, wgrad TN(dy, x)); a GPT-2 `Conv1D` weight (conv1d=True) is
    [in, out] (forward NN, dgrad NT, wgrad TN(x, dy))."""

    def __init__(self, weight, weight_grad=None, bias=None, bias_grad=None, conv1d=False):
        self.weight, self.weight_grad, self.bias, self.bias_grad = weight, weight_grad, bias, bias_grad
        self.conv1d = conv1d

    @classmethod
    def of(cls, weight, bias=None, conv1d=False):
        """Over parameters bound to the flat buffers (.main_grad, if any, is the gradient view)."""
        grad = lambda p: getattr(p, "main_grad", None)
        return cls(weight.data, grad(weight), None if bias is None else bias.data, None if bias is None else grad(bias), conv1d)

    @classmethod
    def span(cls, flat, first, rows, cols, first_bias=None):
        """The [rows, cols] weight starting at parameter `first` and covering the adjacent ones after it; first_bias: the same
        for the bias, a [1, rows] span (the kernels read its `rows` contiguous elements)."""
        return cls(flat.span(first, rows, cols), flat.span(first, rows, cols, grad=True),
                   None if first_bias is None else flat.span(first_bias, 1, rows),
                   None if first_bias is None else flat.span(first_bias, 1, rows, grad=True))

    def __call__(self, x, epilogue=L.EPI_NONE, aux=None):
        return ops.gemm(L.GEMM_NN if self.conv1d else L.GEMM_NT, x, self.weight, bias=self.bias, epilogue=epilogue, aux=aux)

    def forward(self, x, save, epilogue=L.EPI_NONE, aux=None):
        """-> (the output, what backward reads of the input: x itself when `save`, else None). epilogue / aux as __call__."""
        return self(x, epilogue, aux), (x if save else None)

    def saved_input(self, x):
        """What backward reads of the input x, without the GEMM: what forward(x, save=True) returns second."""
        return x

    def backward(self, dy, x, accumulate, dx=None, dx_accumulate=False, colsum=True):
        """-> the gradient of the input x, given dy, the gradient of the output. Writes the weight's gradient (and the bias's)
        into the flat gradient buffer, adding to it when `accumulate`. dx: write the input gradient into this buffer instead,
        adding to it when dx_accumulate. colsum=False: the bias gradient is already written (ops.act_bwd_bias)."""
        if self.conv1d:
            dx = ops.gemm(L.GEMM_NT, dy, self.weight, out=dx, accumulate=dx_accumulate)
            ops.gemm(L.GEMM_TN, x, dy, out=self.weight_grad, accumulate=accumulate)
        else:
            dx = ops.gemm(L.GEMM_NN, dy, self.weight, out=dx, accumulate=dx_accumulate)
            ops.gemm(L.GEMM_TN, dy, x, out=self.weight_grad, accumulate=accumulate)
        if self.bias is not None and colsum:
            ops.colsum(dy, self.bias_grad, accumulate=accumulate)
        return dx


def residual_norm_bwd(dy, x, weight, bias, stats, drop, accumulate, dres=None):
    """Backward of a norm over the sum of a residual and a branch dropped by `drop` (LayerNorm; RMSNorm when `bias` is
    None): -> (gradient of the sum, gradient of the dropped branch), the same tensor when `drop` is None. Writes the
    parameters' gradients into their .main_grad, adding to them when `accumulate`; dres is added to the sum's gradient."""
    if bias is None:
        if drop is None:
            d = ops.rmsnorm_bwd(dy, x, weight.data, stats, weight.main_grad, accumulate=accumulate, dres=dres)
            return d, d
        return ops.rmsnorm_bwd_dropout(dy, x, weight.data, stats, weight.main_grad, drop, accumulate=accumulate, dres=dres)
    if drop is None:
        d = ops.layernorm_bwd(dy, x, weight.data, stats, weight.main_grad, bias.main_grad, accumulate=accumulate, dres=dres)
        return d, d
    return ops.layernorm_bwd_dropout(dy, x, weight.data, stats, weight.main_grad, bias.main_grad, drop, accumulate=accumulate,
                                     dres=dres)


def apply_dropout(x, drop):
    """x through the standalone dropout site `drop` (forward and backward alike); x itself when drop is None."""
    return x if drop is None else ops.dropout(x, drop)


class GatedMLP:
    """m = wo(act(gate) * up) with [gate | up] = wi(h): wi is one projection over the adjacent gate and up weights, `act` the
    gate's activation (L.ACT_SILU for LLaMA, L.ACT_GELU_TANH for mT5). wi and wo are Linear or Fp8Linear."""

    def __init__(self, wi, wo, act):
        self.wi, self.wo, self.act = wi, wo, act

    def __call__(self, h, save=True, drop=None, out=True):
        """-> (m, what the backward reads; with save=False, only what a forward needs is computed). drop: optional
        ops.Dropout on act(gate) * up, the input of wo (mT5's dropout inside the FFN). out=False (with save): stop before
        wo's GEMM, for a recompute whose m nothing reads; m is then None."""
        gu, hs = self.wi.forward(h, save)
        f = gu.shape[1] // 2
        act = ops.glu_fwd(self.act, gu[:, :f], gu[:, f:], drop=drop)
        if not out:
            return None, (hs, gu, self.wo.saved_input(act))
        m, acts = self.wo.forward(act, save)
        return m, (hs, gu, acts)

    def backward(self, dm, saved, accumulate, drop=None):
        """-> the gradient of h; writes the weight gradients as Linear.backward does. drop: the forward's Dropout."""
        hs, gu, act = saved
        f = gu.shape[1] // 2
        dact = self.wo.backward(dm, act, accumulate)
        dgu = torch.empty_like(gu)
        ops.glu_bwd(self.act, dact, gu[:, :f], gu[:, f:], dgu[:, :f], dgu[:, f:], drop=drop)
        return self.wi.backward(dgu, hs, accumulate)


class Fp8Linear:
    """A Linear (HF layout, with or without a bias) run in FP8 with just-in-time per-tensor scaling, with Linear's call
    surface. The weight, the bias and their gradients stay the bf16 flat-buffer views of `lin`; the weight is cast on every
    call, so nothing goes stale after an optimizer step.
      forward: y = x W^T (+ bias, epilogue, aux as Linear) from x e4m3 and W e4m3, both row-major; when saving, x's transposed
               codes and scale are kept for the weight gradient instead of x.
      backward: dy e5m2 (both layouts) and W e4m3 (transposed): dx = dy (W^T)^T, dW (+)= dy^T (x^T)^T into the flat gradient;
                the bias gradient is the bf16 column sum of dy, as Linear's.
    The token count and both extents of W must be multiples of 16."""

    def __init__(self, lin):
        if lin.conv1d:
            raise ValueError("fsb200 Fp8Linear: only [out, in] projections run in FP8 (a Conv1D weight is [in, out])")
        self.lin = lin

    @property
    def bias_grad(self):
        return self.lin.bias_grad

    def __call__(self, x, epilogue=L.EPI_NONE, aux=None):
        return self.forward(x, False, epilogue, aux)[0]

    @staticmethod
    def quantize_input(x, save):
        """x's e4m3 codes as forward makes them: (row-major codes, transposed codes when `save` else None, scale). Projections
        that read the same x (mT5's cross-attention k|v over the encoder output) quantise it once and pass these as `codes`."""
        return ops.fp8_quantize(x, "e4m3", rowwise=True, colwise=save)

    def forward(self, x, save, epilogue=L.EPI_NONE, aux=None, codes=None):
        """codes: quantize_input(x, save), made once for several projections; x is then not read."""
        xq, xt, sx = self.quantize_input(x, save) if codes is None else codes
        wq, sw = self._forward_weight()
        # a bias-free projection without an epilogue (LLaMA's) makes the plain call it made before the epilogue existed
        epi = {} if self.lin.bias is None and epilogue == L.EPI_NONE and aux is None else \
            dict(bias=self.lin.bias, epilogue=epilogue, aux=aux)
        return ops.gemm_fp8(xq, sx, wq, sw, **epi), ((xt, sx) if save else None)

    def saved_input(self, x):
        """What backward reads of the input x, without the GEMM: x's transposed e4m3 codes and scale, the bits forward(x,
        save=True) keeps (the scale depends on x's amax alone, and the cast writes both layouts independently)."""
        _, xt, sx = ops.fp8_quantize(x, "e4m3", rowwise=False, colwise=True)
        return xt, sx

    def backward(self, dy, saved, accumulate, dx=None, dx_accumulate=False, colsum=True):
        """As Linear.backward, with `saved` what forward / saved_input returned."""
        xt, sx = saved
        dyq, dyt, sdy = ops.fp8_quantize(dy, "e5m2", rowwise=True, colwise=True)
        wt, sw = self._dgrad_weight()
        dx = ops.gemm_fp8(dyq, sdy, wt, sw, out=dx, accumulate=dx_accumulate)
        self._wgrad(dyt, sdy, xt, sx, accumulate)
        if self.lin.bias is not None and colsum:
            ops.colsum(dy, self.lin.bias_grad, accumulate=accumulate)
        return dx

    # the weight's layout: the forward's B operand [out, in], the data gradient's [in, out], and the weight gradient's store
    def _forward_weight(self):
        wq, _, sw = ops.fp8_quantize(self.lin.weight, "e4m3")
        return wq, sw

    def _dgrad_weight(self):
        _, wt, sw = ops.fp8_quantize(self.lin.weight, "e4m3", rowwise=False, colwise=True)
        return wt, sw

    def _wgrad(self, dyt, sdy, xt, sx, accumulate):
        ops.gemm_fp8(dyt, sdy, xt, sx, out=self.lin.weight_grad, accumulate=accumulate)


class Fp8Conv1D(Fp8Linear):
    """A GPT-2 Conv1D (Linear(..., conv1d=True): weight [in, out], with or without a bias) in FP8: Fp8Linear's recipe, call
    surface and saved codes, over the other weight layout.
      forward: y = x W (+ bias, epilogue, aux) from x e4m3 row-major and W's transposed e4m3 codes (W^T [out, in]).
      backward: dx = dy W^T from dy e5m2 row-major and W's row-major e4m3 codes; dW (+)= x^T dy written [in, out] into the flat
                gradient by gemm_fp8(store_transposed=True) from dy^T e5m2 and x^T e4m3 codes (the FP8 GEMM takes (e5m2, e4m3) only, so it
                computes dW^T = dy^T x and stores it transposed).
    The same Conv1D as an Fp8Linear over W^T gives the same bits: y, dx and the bias gradient equal, dW its transpose.
    The token count and both extents of W must be multiples of 16."""

    def __init__(self, lin):
        if not lin.conv1d:
            raise ValueError("fsb200 Fp8Conv1D: only [in, out] Conv1D projections (an [out, in] Linear runs as Fp8Linear)")
        self.lin = lin

    def _forward_weight(self):
        return Fp8Linear._dgrad_weight(self)

    def _dgrad_weight(self):
        return Fp8Linear._forward_weight(self)

    def _wgrad(self, dyt, sdy, xt, sx, accumulate):
        ops.gemm_fp8(dyt, sdy, xt, sx, out=self.lin.weight_grad, accumulate=accumulate, store_transposed=True)


# weight format -> (quantiser, (q dtype, q shape, s dtype, s shape) of an [n, k] weight)
WQ = {
    "int8": (ops.quantize_w8, lambda n, k: (torch.int8, (n, k), torch.float32, (n,))),
    "int4": (ops.quantize_w4, lambda n, k: (torch.uint8, (n // 2, k), torch.bfloat16, (n, k // 128))),
}


def quantized_unsupported(model, fmt, what):
    """The error an int8 / int4 model (`model` names its class) raises for `what`."""
    return NotImplementedError(f"fsb200 {model}: {what} is not implemented for an {fmt} (load_in_{fmt[3:]}bit=True) "
                               "model; it only runs inference")


class QuantizedLinear:
    """A layer projection of an int8 / int4 model, with Linear's call surface: the [n, k] weight held as q + scales s in the
    format's layout (WQ) and run through the W8A16 / W4A16 GEMM, with an optional bf16 bias [n] (GPT-2's Conv1D; bias and
    epilogue then run in the GEMM's epilogue). Inference only: saving inputs for a backward, aux and backward raise.
    `model` names the owning class in those errors."""

    def __init__(self, fmt, n, k, device, bias=None, model="model"):
        qd, qs, sd, ss = WQ[fmt][1](n, k)
        self.fmt, self.model = fmt, model
        self.q, self.s = torch.zeros(qs, dtype=qd, device=device), torch.zeros(ss, dtype=sd, device=device)
        self.bias = bias

    def __call__(self, x, epilogue=L.EPI_NONE):
        gemm = ops.gemm_w8a16 if self.fmt == "int8" else ops.gemm_w4a16
        if self.bias is None and epilogue == L.EPI_NONE:   # LLaMA's projections: the bias-free call
            return gemm(x, self.q, self.s)
        return gemm(x, self.q, self.s, bias=self.bias, epilogue=epilogue)

    def forward(self, x, save, epilogue=L.EPI_NONE, aux=None):
        if save or aux is not None:
            raise quantized_unsupported(self.model, self.fmt, "a forward that keeps activations for a backward")
        return self(x, epilogue), None

    def backward(self, *_, **__):
        raise quantized_unsupported(self.model, self.fmt, "backward")
