"""CPU restatement of the NF4 weight format (load_4bit) — TEST INFRASTRUCTURE ONLY.

The reference loads 4-bit models through bitsandbytes (llava/model/builder.py:26-41: load_in_4bit, quant_type "nf4",
double quantisation, fp16 compute dtype). bitsandbytes is not part of this package, so this file DEFINES the arithmetic the
CUDA kernels (csrc/nf4.cu) implement. It follows bitsandbytes' NF4 where that costs nothing:

  table          the 16 NF4 values, bitsandbytes' create_normal_map(offset=0.9677083) (restated in `normal_map`)
  quantize_nf4   per row, every block of 64 consecutive K elements: absmax = fp32 max |w|; x = w / absmax (IEEE fp32
                 division); code = number of fp32 midpoints (t[i] + t[i+1]) * 0.5 that x lies STRICTLY above (a value on a
                 midpoint takes the lower code, as bitsandbytes' dQuantizeNF4, which compares with `>`); an all-zero block
                 stores absmax 0 and code 7 (the table's 0.0)
  dequantize_nf4 w_hat = bf16_rn(fp32(table[code]) * absmax)
  layout         codes [N, K/2] bytes, element 2j in the high nibble of byte j (bitsandbytes' order); absmax [N, K/64] fp32.
                 pack_nf4(order="gemv") restates the order the engine keeps for its decode GEMV (csrc/nf4.cu): within each
                 128-element chunk of a row, the 16-bit word of elements 4G .. 4G+3, G = 4m + t, moves to word 8t + m.

Deliberate differences from bitsandbytes (DESIGN.md §2): the absmax stays fp32 (no double quantisation of the absmax to
8 bits per 256 blocks; `bnb_4bit_use_double_quant` is accepted and has no effect), and the compute dtype is bf16.

nf4_weights(w, cfg) gives the oracle weight dict of an NF4 engine: the seven decoder Linears of every layer and both
mm_projector weights replaced by w_hat. Quantisation is per row along K, so the HF matrices can be quantised one by one:
the engine's fused Wqkv (rows q | k | v) and block-64 interleaved gate/up rows hold the same rows.
"""
import torch

BLOCK = 64

# bitsandbytes' NF4 table (functional.py, get_4bit_type("nf4")), as fp32
NF4_TABLE = torch.tensor([
    -1.0, -0.6961928009986877, -0.5250730514526367, -0.39491748809814453, -0.28444138169288635, -0.18477343022823334,
    -0.09105003625154495, 0.0, 0.07958029955625534, 0.16093020141124725, 0.24611230194568634, 0.33791524171829224,
    0.44070982933044434, 0.5626170039176941, 0.7229568362236023, 1.0], dtype=torch.float32)

DECODER_LINEARS = ("self_attn.q_proj.weight", "self_attn.k_proj.weight", "self_attn.v_proj.weight", "self_attn.o_proj.weight",
                   "mlp.gate_proj.weight", "mlp.up_proj.weight", "mlp.down_proj.weight")
PROJECTOR_WEIGHTS = ("model.mm_projector.0.weight", "model.mm_projector.2.weight")


def normal_map(offset=0.9677083):
    """bitsandbytes create_normal_map(offset, use_extra_value=True), reduced to its 16 distinct values: the normal quantiles
    of linspace(offset, 0.5, 9)[:-1], the negated quantiles of linspace(offset, 0.5, 8)[:-1] and 0, sorted, divided by the
    maximum (fp32, as bitsandbytes computes it)."""
    from scipy.stats import norm

    v1 = norm.ppf(torch.linspace(offset, 0.5, 9)[:-1]).tolist()
    v3 = (-norm.ppf(torch.linspace(offset, 0.5, 8)[:-1])).tolist()
    values = torch.tensor(v1 + [0.0] + v3, dtype=torch.float32).sort().values
    return values / values.max()


def midpoints():
    t = NF4_TABLE
    return (t[:-1] + t[1:]) * 0.5  # fp32 add, exact halving


def quantize_nf4(w: torch.Tensor):
    """w [N, K] (values taken as fp32; K % 64 == 0) -> (codes uint8 [N, K] in 0..15, absmax fp32 [N, K/64])."""
    N, K = w.shape
    assert K % BLOCK == 0, K
    wb = w.float().reshape(N, K // BLOCK, BLOCK)
    absmax = wb.abs().amax(dim=-1)
    zero = absmax == 0
    x = wb / torch.where(zero, torch.ones_like(absmax), absmax)[..., None]  # tensor / tensor: IEEE division
    # number of midpoints strictly below x (bucketize with right=False: mid[i-1] < x <= mid[i] -> i)
    codes = torch.bucketize(x, midpoints().to(x.device), right=False).to(torch.uint8)
    codes = torch.where(zero[..., None], torch.full_like(codes, 7), codes)
    return codes.reshape(N, K), absmax


def dequantize_nf4(codes: torch.Tensor, absmax: torch.Tensor):
    """codes uint8 [N, K], absmax [N, K/64] -> w_hat bf16 [N, K]."""
    N, K = codes.shape
    v = NF4_TABLE.to(codes.device)[codes.long()].reshape(N, K // BLOCK, BLOCK) * absmax[..., None]
    return v.reshape(N, K).to(torch.bfloat16)


def w_hat(w: torch.Tensor):
    return dequantize_nf4(*quantize_nf4(w))


def pack_nf4(codes: torch.Tensor, order="canonical"):
    """codes uint8 [N, K] -> bytes [N, K/2]; order "canonical" (element 2j in the high nibble of byte j) or "gemv"."""
    N, K = codes.shape
    b = (codes[:, 0::2] << 4) | codes[:, 1::2]
    if order == "canonical":
        return b.contiguous()
    assert order == "gemv" and K % 128 == 0, (order, K)
    # [N, chunk, m (8), t (4), 2 bytes] -> [N, chunk, t, m, 2]
    return b.reshape(N, K // 128, 8, 4, 2).permute(0, 1, 3, 2, 4).reshape(N, K // 2).contiguous()


def unpack_nf4(packed: torch.Tensor, order="canonical"):
    """Inverse of pack_nf4."""
    N, K2 = packed.shape
    b = packed
    if order == "gemv":
        b = b.reshape(N, K2 // 64, 4, 8, 2).permute(0, 1, 3, 2, 4).reshape(N, K2)
    else:
        assert order == "canonical", order
    out = torch.empty(N, 2 * K2, dtype=torch.uint8, device=packed.device)
    out[:, 0::2] = b >> 4
    out[:, 1::2] = b & 15
    return out


def nf4_weights(w: dict, cfg: dict):
    """Oracle weight dict of an NF4 engine built from `w`: decoder Linears and projector weights replaced by w_hat (in the
    dtype of the input tensor). Returns a NEW dict; other tensors are shared."""
    out = dict(w)
    keys = [f"model.layers.{i}.{k}" for i in range(cfg["layers"]) for k in DECODER_LINEARS] + list(PROJECTOR_WEIGHTS)
    for k in keys:
        if k in w:
            out[k] = w_hat(w[k]).to(w[k].dtype)
    return out


def nf4_linear_bytes(N, K):
    """Device bytes of one NF4 Linear: codes + fp32 absmax."""
    return N * K // 2 + 4 * N * K // BLOCK
