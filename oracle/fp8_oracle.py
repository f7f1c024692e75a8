"""ORACLE -- test infrastructure, not product code.

The FP8 mode (STA(precision="fp8"), include/sta_b200.h STA_PRECISION_FP8) restated on the CPU: StaOracle's bf16 operand
emulation, except that every linear of the 24 encoder and 12 decoder blocks takes e4m3 operands, quantised and
dequantised with the recipe of the kernels:
  * e4m3 "fn" (max 448), round to nearest even, saturating;
  * power-of-two scales s = 2^e, e the smallest integer with amax <= 448 * 2^e (read from the exponent and mantissa
    bits, as the kernels do), s = 1 for an all-zero group, e >= -126;
  * activations: one scale per row and 128 columns; weights: one scale per 128 x 128 block of W [N][K].
The operands are quantised from exactly the tensors the kernels quantise: the fp32 LayerNorm outputs (encoder norm1 /
norm2, decoder norm1 / norm_y / norm2 / norm3), the fp32 GELU output of fc1 and the bf16 attention output.  The products
of the dequantised operands are summed in fp32 by torch, not block by block as on the tensor cores; tests allow for that.
"""
import torch
import torch.nn.functional as F

from oracle.sta_oracle import DEC_HEADS, ENC_DEPTH, ENC_HEADS, StaOracle, rope2d, token_positions

E4M3_MAX = 448.0


def fp8_scale(amax):
    """Power-of-two scales of groups with absolute maxima `amax` (fp32 tensor): (s, 1 / s), both exact."""
    b = amax.to(torch.float32).contiguous().view(torch.int32)
    E = (b >> 23) & 0xFF
    e = E - 135 + ((b & 0x7FFFFF) > 0x600000).to(torch.int32)
    e = torch.where(E == 0, torch.full_like(e, -126), e).clamp(min=-126)
    e = torch.where(b == 0, torch.zeros_like(e), e)
    s = ((e + 127) << 23).view(torch.float32)
    inv = ((127 - e) << 23).view(torch.float32)
    return s, inv


def quantize_rows(x):
    """x [..., C] fp32, C % 128 == 0 -> (e4m3 codes [..., C] as torch.float8_e4m3fn, scales [..., C / 128])."""
    C = x.shape[-1]
    g = x.to(torch.float32).reshape(*x.shape[:-1], C // 128, 128)
    s, inv = fp8_scale(g.abs().amax(-1))
    q = (g * inv[..., None]).clamp(-E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn)
    return q.reshape(x.shape), s


def dequantize_rows(q, s):
    C = q.shape[-1]
    return (q.float().reshape(*q.shape[:-1], C // 128, 128) * s[..., None]).reshape(q.shape)


def quantize_blocks(w):
    """w [N][K] fp32, N and K multiples of 128 -> (e4m3 codes [N][K], scales [N / 128][K / 128])."""
    N, K = w.shape
    g = w.to(torch.float32).reshape(N // 128, 128, K // 128, 128)
    s, inv = fp8_scale(g.abs().amax(dim=(1, 3)))
    q = (g * inv[:, None, :, None]).clamp(-E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn)
    return q.reshape(N, K), s


def dequantize_blocks(q, s):
    N, K = q.shape
    return (q.float().reshape(N // 128, 128, K // 128, 128) * s[:, None, :, None]).reshape(N, K)


def qdq_rows(x):
    return dequantize_rows(*quantize_rows(x))


class Fp8Oracle(StaOracle):
    def __init__(self, state_dict):
        super().__init__(state_dict, emulate_bf16=True)
        self._w8 = {}

    def w8(self, name):
        if name not in self._w8:
            self._w8[name] = dequantize_blocks(*quantize_blocks(self.sd[name]))
        return self._w8[name]

    def lin8(self, xq, prefix):
        """trunk linear on already quantised-dequantised rows"""
        return F.linear(xq, self.w8(prefix + ".weight"), self.p(prefix + ".bias"))

    def mlp8(self, xn, prefix):
        h = F.gelu(self.lin8(qdq_rows(xn), prefix + ".fc1"))  # the fp32 GELU output is quantised
        return self.lin8(qdq_rows(h), prefix + ".fc2")

    def self_attn8(self, xn, pos, prefix, heads):
        B, N, C = xn.shape
        qkv = self.lin8(qdq_rows(xn), prefix + ".qkv").reshape(B, N, 3, heads, C // heads).permute(2, 0, 3, 1, 4)
        q, k, v = self.q(rope2d(qkv[0], pos)), self.q(rope2d(qkv[1], pos)), self.q(qkv[2])
        o = self.q(self.attention(q, k, v).transpose(1, 2).reshape(B, N, C))  # bf16 attention output
        return self.lin8(qdq_rows(o), prefix + ".proj")

    def cross_attn8(self, xn, ynq, xpos, ypos, prefix, heads):
        B, Nq, C = xn.shape
        Nk = ynq.shape[1]
        q = self.lin8(qdq_rows(xn), prefix + ".projq").reshape(B, Nq, heads, C // heads).transpose(1, 2)
        k = self.lin8(ynq, prefix + ".projk").reshape(B, Nk, heads, C // heads).transpose(1, 2)
        v = self.lin8(ynq, prefix + ".projv").reshape(B, Nk, heads, C // heads).transpose(1, 2)
        q, k, v = self.q(rope2d(q, xpos)), self.q(rope2d(k, ypos)), self.q(v)
        o = self.q(self.attention(q, k, v).transpose(1, 2).reshape(B, Nq, C))
        return self.lin8(qdq_rows(o), prefix + ".proj")

    def encode_image(self, img):
        B, _, H, W = img.shape
        h, w = H // 16, W // 16
        x = F.conv2d(self.q(img.to(torch.float32)), self.w("patch_embed.proj.weight"), self.p("patch_embed.proj.bias"),
                     stride=16)
        x = x.flatten(2).transpose(1, 2)
        pos = token_positions(B, h, w)
        for i in range(ENC_DEPTH):
            p = "enc_blocks.%d" % i
            x = x + self.self_attn8(self.ln(x, p + ".norm1"), pos, p + ".attn", ENC_HEADS)
            x = x + self.mlp8(self.ln(x, p + ".norm2"), p + ".mlp")
        return x, pos

    def dec_block(self, x, y, xpos, ypos, i):
        p = "dec_block.%d" % i
        x = x + self.self_attn8(self.ln(x, p + ".norm1"), xpos, p + ".attn", DEC_HEADS)
        ynq = qdq_rows(self.ln(y, p + ".norm_y"))
        x = x + self.cross_attn8(self.ln(x, p + ".norm2"), ynq, xpos, ypos, p + ".cross_attn", DEC_HEADS)
        x = x + self.mlp8(self.ln(x, p + ".norm3"), p + ".mlp")
        return x

