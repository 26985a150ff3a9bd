"""Drop-in for model/networks/resample2d_package/resample2d.py."""
import torch
from torch.autograd import Function
from torch.nn.modules.module import Module

from . import functional as F_


class Resample2dFunction(Function):
    """reference: resample2d.py:6-39.  input2 carries (dx, dy, sigma)."""

    @staticmethod
    def forward(ctx, input1, input2, kernel_size=2, dilation=1):
        assert input1.is_contiguous()
        assert input2.is_contiguous()
        ctx.save_for_backward(input1, input2)
        ctx.kernel_size = kernel_size
        ctx.dilation = dilation
        return F_.resample2d_fwd(input1, input2, kernel_size, dilation)

    @staticmethod
    def backward(ctx, grad_output):
        input1, input2 = ctx.saved_tensors
        grad_input1, grad_input2 = F_.resample2d_bwd(input1, input2, grad_output, ctx.kernel_size, ctx.dilation)
        return grad_input1, grad_input2.to(input2.dtype), None, None


class Resample2d(Module):
    """reference: resample2d.py:41-53.

    One deliberate difference: the reference builds ``self.sigma`` with
    ``.cuda()`` inside ``__init__`` (resample2d.py:47), which needs a GPU at
    construction time and pins the module to device 0; here sigma is kept as a
    Python float and materialised on the input's device in ``forward``.

    bf16 / fp16 ``input1`` runs on the 16-bit kernels with an fp32 flow (a 16-bit flow is widened, and so is one next
    to an fp32 ``input1``): the output has ``input1``'s dtype, each gradient the dtype of its own input."""

    def __init__(self, kernel_size=2, dilation=1, sigma=5):
        super(Resample2d, self).__init__()
        self.kernel_size = kernel_size
        self.dilation = dilation
        self.sigma = float(sigma)

    def forward(self, input1, input2):
        input1_c = input1.contiguous()
        input2 = F_.flow_f32(input1_c, input2)            # the sigma plane is built in the dtype the kernels read
        sigma = torch.full((input2.size(0), 1, input2.size(2), input2.size(3)), self.sigma,
                           dtype=input2.dtype, device=input2.device)
        input2 = torch.cat((input2, sigma), 1)
        return Resample2dFunction.apply(input1_c, input2, self.kernel_size, self.dilation)


class Resample2dCosineFunction(Function):
    """cosine_similarity(Resample2dFunction(input1, input2), target, dim=1, eps) as ONE op each way (SURVEY row f4;
    external_function.py:275-279).  The warped tensor is neither written nor saved: the backward rebuilds each channel of it
    in registers.  Gradients are produced only for the inputs that ask for one -- in the reference's loss that is the flow."""

    @staticmethod
    def forward(ctx, input1, input2, target, kernel_size=2, dilation=1, eps=1e-8):
        assert input1.is_contiguous()
        assert input2.is_contiguous()
        target = target.contiguous()
        cos, stats = F_.resample2d_cosine_fwd(input1, input2, target, kernel_size, dilation, eps)
        ctx.save_for_backward(input1, input2, target, stats)
        ctx.cfg = (kernel_size, dilation, eps)
        return cos

    @staticmethod
    def backward(ctx, grad_cos):
        input1, input2, target, stats = ctx.saved_tensors
        ks, dil, eps = ctx.cfg
        g1, g2, gt = F_.resample2d_cosine_bwd(input1, input2, target, stats, grad_cos, ks, dil, eps,
                                              need_input1=ctx.needs_input_grad[0], need_target=ctx.needs_input_grad[2])
        return g1, g2.to(input2.dtype), gt, None, None, None


class Resample2dCosine(Module):
    """``Resample2dCosine(ks, dil, sigma)(source, flow, target)`` == ``F.cosine_similarity(Resample2d(ks, dil, sigma)(source, flow),
    target)`` -> [B,H,W]."""

    def __init__(self, kernel_size=2, dilation=1, sigma=5, eps=1e-8):
        super(Resample2dCosine, self).__init__()
        self.kernel_size = kernel_size
        self.dilation = dilation
        self.sigma = float(sigma)
        self.eps = float(eps)

    def forward(self, input1, input2, target):
        input2 = F_.flow_f32(input1, input2)
        sigma = torch.full((input2.size(0), 1, input2.size(2), input2.size(3)), self.sigma, dtype=input2.dtype, device=input2.device)
        input2 = torch.cat((input2, sigma), 1)
        return Resample2dCosineFunction.apply(input1.contiguous(), input2, target, self.kernel_size, self.dilation, self.eps)
