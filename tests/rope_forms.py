"""The two ways Llama code writes RoPE, and the test-local Llama variants that use them: the
half-split form of workloads._rope and the rotate_half form of the Hugging Face Llama."""
import torch
import torch.nn.functional as F

from easydist_b200 import workloads

FORMS = ["half_split", "rotate_half"]


def rope_half_split(x, cos, sin):
    return workloads._rope(x, cos, sin)


def rope_rotate_half(x, cos, sin):
    h = x.shape[-1] // 2
    c, s = torch.cat((cos, cos), -1), torch.cat((sin, sin), -1)
    return x * c + torch.cat((-x[..., h:], x[..., :h]), -1) * s


def _rope_promoted(x, cos, sin):
    """The half-split form with fp32 tables: the products are promoted to fp32."""
    return workloads._rope(x, cos.float(), sin.float()).to(x.dtype)


class _Block(workloads.LlamaBlock):
    """workloads.LlamaBlock.forward with another RoPE function (same parameters)."""
    rope_fn = None

    def forward(self, x, cos, sin):
        B, T, C = x.shape
        h = self.ln1(x)
        q, k, v = (w(h).view(B, T, self.n_head, C // self.n_head).transpose(1, 2)
                   for w in (self.wq, self.wk, self.wv))
        rope = type(self).rope_fn
        y = F.scaled_dot_product_attention(rope(q, cos, sin), rope(k, cos, sin), v, is_causal=True)
        x = x + self.wo(y.transpose(1, 2).contiguous().view(B, T, C))
        h = self.ln2(x)
        return x + self.w_down(F.silu(self.w_gate(h)) * self.w_up(h))


class RotateHalfBlock(_Block):
    rope_fn = staticmethod(rope_rotate_half)


class PromotedTableBlock(_Block):
    rope_fn = staticmethod(_rope_promoted)


def llama(cfg, form="half_split"):
    """workloads.Llama with its RoPE written in `form` ("half_split", "rotate_half" or
    "promoted_table")."""
    m = workloads.Llama(cfg)
    cls = {"half_split": None, "rotate_half": RotateHalfBlock, "promoted_table": PromotedTableBlock}[form]
    if cls is not None:
        for blk in m.h:
            blk.__class__ = cls
    return m


def tables(T, hd, dtype, device="cpu"):
    inv = 1.0 / (10000.0 ** (torch.arange(0, hd, 2, device=device).float() / hd))
    ang = torch.arange(T, device=device).float()[:, None] * inv[None, :]
    return ang.cos().to(dtype), ang.sin().to(dtype)
