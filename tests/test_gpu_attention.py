"""`precondition_attention` on the GPU:

  * the strided entry points (kfac_factor_linear_strided, kfac_rows_linear_strided, kfac_reduce_rows_linear_strided)
    give the bits of the existing entry points at ld == features and on a contiguous copy of a column block; the
    sequence-first reduce matches fp64;
  * stock attention blocks (nn.TransformerEncoderLayer with batch_first both ways, nn.TransformerDecoderLayer with its
    cross-attention, a ViT-style block) against their twin -- the same block written with four nn.Linear layers and
    F.scaled_dot_product_attention, weights copied -- under EIGEN / INVERSE / EKFAC, expand / reduce, fp16 autocast with
    a GradScaler, accumulation_steps=2 and a factor/inverse schedule: per-projection A and G agree to 1e-5
    rel-Frobenius, every preconditioned gradient to 1e-3;
  * a skipped projection keeps its raw gradient rows bit for bit;
  * the reference language-model example's configuration with every layer preconditioned trains;
  * two ranks (tests/dist_attention.py): COMM_OPT and MEM_OPT, eigen and inverse, bit-identical gradients on every
    rank, fp64 on the concatenated batch, the twin model's collectives.
Gradients are compared under the math SDPA backend (the flash backward need not be deterministic).
"""
import copy

import pytest
import torch
import torch.nn.functional as F
from torch import nn
from torch.nn.attention import SDPBackend, sdpa_kernel

from conftest import rel_fro

pytestmark = pytest.mark.gpu

DEV = torch.device('cuda')


@pytest.fixture(scope='module')
def lib():
    from kfac_b200 import _cabi
    return _cabi.load()


def S():
    return torch.cuda.current_stream().cuda_stream


def _code(dtype):
    from kfac_b200 import _cabi
    return _cabi.DTYPE_CODE[dtype]


# ---------------------------------------------------------------------------------------------- kernels
def _factor(lib, x, rows, F_, ld, ones, strided):
    d = F_ + ones
    acc = torch.zeros(d, d, device=DEV)
    if strided:
        need = lib.kfac_factor_linear_strided_workspace_bytes(rows, F_, ld, ones)
        ws = torch.empty(max(need, 1), dtype=torch.uint8, device=DEV)
        rc = lib.kfac_factor_linear_strided(x.data_ptr(), _code(x.dtype), rows, F_, ld, ones, 0.5, acc.data_ptr(),
                                            ws.data_ptr(), need, S())
    else:
        need = lib.kfac_factor_linear_workspace_bytes(rows, F_, ones)
        ws = torch.empty(max(need, 1), dtype=torch.uint8, device=DEV)
        rc = lib.kfac_factor_linear(x.data_ptr(), _code(x.dtype), rows, F_, ones, 0.5, acc.data_ptr(), ws.data_ptr(),
                                    need, S())
    assert rc == 0, lib.kfac_last_error()
    return acc


@pytest.mark.parametrize('dtype', [torch.float32, torch.float16, torch.bfloat16])
@pytest.mark.parametrize('rows,F_', [(40, 24), (1024, 192), (4096, 64)])
@pytest.mark.parametrize('ones', [0, 1])
def test_factor_linear_strided(lib, dtype, rows, F_, ones):
    torch.manual_seed(0)
    x = torch.randn(rows, 3 * F_, device=DEV).to(dtype)
    blk = x[:, F_:2 * F_]
    a = _factor(lib, blk, rows, F_, 3 * F_, ones, True)
    b = _factor(lib, blk.contiguous(), rows, F_, F_, ones, False)
    full_s = _factor(lib, x, rows, 3 * F_, 3 * F_, ones, True)
    full = _factor(lib, x, rows, 3 * F_, 3 * F_, ones, False)
    torch.cuda.synchronize()
    assert torch.equal(a, b) and torch.equal(full_s, full)
    ref = 0.5 * blk.double().T @ blk.double()
    assert rel_fro(a[:F_, :F_], ref) < 1e-5


@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16])
@pytest.mark.parametrize('ones', [0, 1])
def test_rows_linear_strided(lib, dtype, ones):
    torch.manual_seed(1)
    rows, F_ = 300, 40
    x = torch.randn(rows, 3 * F_, device=DEV).to(dtype)
    ls = torch.tensor([4.0], device=DEV)
    ld = (F_ + ones + 3) // 4 * 4
    outs = []
    for ptr, ldx, call in ((x[:, 2 * F_:].data_ptr(), 3 * F_, 'strided'), (x[:, 2 * F_:].contiguous(), F_, 'plain')):
        out = torch.full((rows, ld), float('nan'), device=DEV)
        if call == 'strided':
            rc = lib.kfac_rows_linear_strided(ptr, _code(dtype), rows, F_, ldx, ones, 0.5, ls.data_ptr(),
                                              out.data_ptr(), ld, S())
        else:
            rc = lib.kfac_rows_linear(ptr.data_ptr(), _code(dtype), rows, F_, ones, 0.5, ls.data_ptr(), out.data_ptr(),
                                      ld, S())
        assert rc == 0, lib.kfac_last_error()
        outs.append(out)
    torch.cuda.synchronize()
    assert torch.equal(outs[0], outs[1])


@pytest.mark.parametrize('dtype', [torch.float32, torch.float16])
@pytest.mark.parametrize('R,B,F_', [(128, 8, 96), (5, 3, 40), (1000, 2, 33)])
def test_reduce_rows_linear_strided(lib, dtype, R, B, F_):
    torch.manual_seed(2)
    x = torch.randn(R, B, 3 * F_, device=DEV).to(dtype)          # sequence-first packed projection
    blk = x[..., F_:2 * F_]
    ld = F_ + 1

    def run(ptr, sb, st):
        out = torch.full((B, ld), float('nan'), device=DEV)
        rc = lib.kfac_reduce_rows_linear_strided(ptr, _code(dtype), B, R, F_, sb, st, 1, 0.25, None, out.data_ptr(),
                                                 ld, S())
        assert rc == 0, lib.kfac_last_error()
        return out

    a = run(blk.data_ptr(), 3 * F_, B * 3 * F_)
    c = blk.transpose(0, 1).contiguous()                          # (B, R, F) contiguous copy
    b = torch.full((B, ld), float('nan'), device=DEV)
    assert lib.kfac_reduce_rows_linear(c.data_ptr(), _code(dtype), B, R, F_, 1, 0.25, None, b.data_ptr(), ld, S()) == 0
    b2 = run(c.data_ptr(), R * F_, F_)
    torch.cuda.synchronize()
    assert torch.equal(a, b) and torch.equal(b2, b)
    ref = 0.25 * blk.double().sum(0)
    assert rel_fro(a[:, :F_], ref) < 1e-6
    assert torch.all(a[:, F_] == 0.25 * R)


# ---------------------------------------------------------------------------------------------- twins
class TwinAttention(nn.Module):
    """The same attention with four nn.Linear layers and F.scaled_dot_product_attention, weights copied."""

    def __init__(self, m: nn.MultiheadAttention):
        super().__init__()
        E, bias = m.embed_dim, m.in_proj_bias is not None
        self.H, self.batch_first = m.num_heads, m.batch_first
        self.q_proj = nn.Linear(E, E, bias=bias)
        self.k_proj = nn.Linear(m.kdim, E, bias=bias)
        self.v_proj = nn.Linear(m.vdim, E, bias=bias)
        self.out_proj = nn.Linear(E, E, bias=m.out_proj.bias is not None)
        with torch.no_grad():
            for i, lin in enumerate((self.q_proj, self.k_proj, self.v_proj)):
                w = m.in_proj_weight[i * E:(i + 1) * E] if m._qkv_same_embed_dim else getattr(m, 'qkv'[i] + '_proj_weight')
                lin.weight.copy_(w)
                if bias:
                    lin.bias.copy_(m.in_proj_bias[i * E:(i + 1) * E])
            self.out_proj.weight.copy_(m.out_proj.weight)
            if m.out_proj.bias is not None:
                self.out_proj.bias.copy_(m.out_proj.bias)

    def forward(self, query, key, value, key_padding_mask=None, need_weights=False, attn_mask=None,
                average_attn_weights=True, is_causal=False):
        if not self.batch_first:
            query, key, value = (t.transpose(0, 1) for t in (query, key, value))
        B, L, E = query.shape
        Sn = key.size(1)
        h = lambda t, n: t.view(B, n, self.H, E // self.H).transpose(1, 2)  # noqa: E731
        q, k, v = h(self.q_proj(query), L), h(self.k_proj(key), Sn), h(self.v_proj(value), Sn)
        mask = None
        if attn_mask is not None:
            mask = attn_mask if attn_mask.dtype != torch.bool else torch.zeros_like(attn_mask, dtype=q.dtype).masked_fill(
                attn_mask, float('-inf'))
        if key_padding_mask is not None:
            kpm = torch.zeros(B, 1, 1, Sn, device=q.device, dtype=q.dtype).masked_fill(
                key_padding_mask.view(B, 1, 1, Sn), float('-inf'))
            mask = kpm if mask is None else mask + kpm
        o = F.scaled_dot_product_attention(q, k, v, attn_mask=mask, is_causal=is_causal and mask is None)
        o = self.out_proj(o.transpose(1, 2).reshape(B, L, E))
        return (o if self.batch_first else o.transpose(0, 1)), None


def _twin(model):
    twin = copy.deepcopy(model)
    for name, m in list(twin.named_modules()):
        for cname, c in list(m.named_children()):
            if isinstance(c, nn.MultiheadAttention):
                setattr(m, cname, TwinAttention(c).to(c.in_proj_weight.device))
    return twin


class Enc(nn.Module):
    def __init__(self, batch_first):
        super().__init__()
        self.layer = nn.TransformerEncoderLayer(64, 4, 128, dropout=0.0, batch_first=batch_first)
        self.head = nn.Linear(64, 10)
        self.batch_first = batch_first

    def forward(self, x):
        if self.batch_first:
            return self.head(self.layer(x))
        return self.head(self.layer(x.transpose(0, 1))).transpose(0, 1)


class Dec(nn.Module):
    def __init__(self):
        super().__init__()
        self.mem = nn.Linear(32, 64)
        self.layer = nn.TransformerDecoderLayer(64, 4, 128, dropout=0.0, batch_first=True)
        self.head = nn.Linear(64, 10)

    def forward(self, x):
        return self.head(self.layer(x, self.mem(x[:, :6, :32])))


class ViTBlock(nn.Module):
    def __init__(self):
        super().__init__()
        self.ln_1 = nn.LayerNorm(64)
        self.self_attention = nn.MultiheadAttention(64, 4, batch_first=True)
        self.mlp = nn.Sequential(nn.Linear(64, 128), nn.GELU(), nn.Linear(128, 64))
        self.head = nn.Linear(64, 10)

    def forward(self, x):
        y = self.ln_1(x)
        y, _ = self.self_attention(y, y, y, need_weights=False)
        x = x + y
        return self.head(x + self.mlp(x))


MODELS = {'enc_bf': lambda: Enc(True), 'enc_sf': lambda: Enc(False), 'dec': Dec, 'vit': ViTBlock}


def _grads(model):
    """name -> (out, in + 1) gradient matrix [W | b] of every Linear-equivalent layer, the attention projections split
    out of in_proj_weight / in_proj_bias.  (The whole matrix, as the layer preconditions it: the key bias alone has a
    gradient of rounding noise only, softmax being invariant to it.)"""
    out = {}
    for name, m in model.named_modules():
        if isinstance(m, nn.MultiheadAttention):
            E = m.embed_dim
            for i, w in enumerate('qkv'):
                out[f'{name}.{w}_proj'] = torch.cat([m.in_proj_weight.grad[i * E:(i + 1) * E],
                                                     m.in_proj_bias.grad[i * E:(i + 1) * E, None]], 1)
        elif isinstance(m, nn.Linear):
            out[name] = torch.cat([m.weight.grad, m.bias.grad[:, None]], 1)
    return out


def _run(model, kw, steps, batches, amp=False, accum=1):
    """`steps` preconditioner steps on fixed weights (the two models stay on the same point); the preconditioned
    gradients of every step."""
    from kfac_b200.preconditioner import KFACPreconditioner
    scaler = torch.amp.GradScaler('cuda', init_scale=2.0 ** 10) if amp else None
    opt = torch.optim.SGD(model.parameters(), lr=0.0)
    pre = KFACPreconditioner(model, damping=0.01, factor_decay=0.9, lr=0.1, grad_scaler=scaler,
                             accumulation_steps=accum, **kw)
    tgt = torch.randn(batches[0].shape[0], batches[0].shape[1], 10, device=DEV,
                      generator=torch.Generator(DEV).manual_seed(9))
    grads = []
    for s in range(steps):
        opt.zero_grad()
        for a in range(accum):
            x = batches[(s * accum + a) % len(batches)]
            with torch.autocast('cuda', dtype=torch.float16, enabled=amp):
                loss = (model(x).float() - tgt).pow(2).mean() / accum
            (scaler.scale(loss) if amp else loss).backward()
        if amp:
            scaler.unscale_(opt)
        pre.step()
        grads.append({k: v.detach().clone() for k, v in _grads(model).items()})
        if amp:
            scaler.step(opt)
            scaler.update()
    return pre, grads


CONFIGS = [
    ('enc_bf', dict(compute_method='eigen')), ('enc_sf', dict(compute_method='eigen')),
    ('dec', dict(compute_method='eigen')), ('vit', dict(compute_method='eigen')),
    ('enc_bf', dict(compute_method='inverse')), ('dec', dict(compute_method='inverse')),
    ('enc_bf', dict(compute_method='ekfac')), ('vit', dict(compute_method='ekfac')),
    ('enc_bf', dict(compute_method='eigen', kfac_approx='reduce')),
    ('enc_sf', dict(compute_method='inverse', kfac_approx='reduce')),
    ('dec', dict(compute_method='ekfac', kfac_approx='reduce')),
    ('enc_bf', dict(compute_method='eigen', amp=True)), ('vit', dict(compute_method='inverse', amp=True)),
    ('dec', dict(compute_method='eigen', accum=2)),
    ('vit', dict(compute_method='eigen', factor_update_steps=2, inv_update_steps=4)),
]


@pytest.mark.parametrize('model_name,cfg', CONFIGS, ids=[f'{m}-{"-".join(f"{k}={v}" for k, v in c.items())}'
                                                          for m, c in CONFIGS])
def test_against_twin(model_name, cfg):
    cfg = dict(cfg)
    amp, accum = cfg.pop('amp', False), cfg.pop('accum', 1)
    torch.manual_seed(0)
    model = MODELS[model_name]().to(DEV)
    twin = _twin(model)
    g = torch.Generator(DEV).manual_seed(1)
    batches = [torch.randn(8, 12, 64, device=DEV, generator=g) for _ in range(4)]
    steps = 5
    with sdpa_kernel(SDPBackend.MATH):
        pre, got = _run(model, dict(precondition_attention=True, **cfg), steps, batches, amp, accum)
        tpre, want = _run(twin, cfg, steps, batches, amp, accum)
    mine = {n: l for n, l in pre._layers.values()}
    theirs = {n: l for n, l in tpre._layers.values()}
    assert mine.keys() == theirs.keys()
    assert sum(n.endswith('_proj') for n in mine) >= 4
    for n in mine:
        for side in ('a_factor', 'g_factor'):
            assert rel_fro(getattr(mine[n], side), getattr(theirs[n], side)) <= 1e-5, (n, side)
    for s in range(steps):
        for k in want[s]:
            assert rel_fro(got[s][k], want[s][k]) <= 1e-3, (s, k)
    assert pre.memory_usage() == tpre.memory_usage()
    assert {n: (v['A'].shape, v['G'].shape) for n, v in pre.state_dict()['layers'].items()} == \
        {n: (v['A'].shape, v['G'].shape) for n, v in tpre.state_dict()['layers'].items()}


def test_skipped_projection_keeps_raw_gradient():
    from kfac_b200.preconditioner import KFACPreconditioner
    torch.manual_seed(0)
    model = Enc(True).to(DEV)
    pre = KFACPreconditioner(model, precondition_attention=True, skip_layers=[r'k_proj'], damping=0.01)
    assert 'layer.self_attn.k_proj' not in [n for n, _ in pre._layers.values()]
    x = torch.randn(4, 12, 64, device=DEV)
    for _ in range(2):
        model.zero_grad()
        model(x).pow(2).mean().backward()
        raw = model.layer.self_attn.in_proj_weight.grad.clone()
        rawb = model.layer.self_attn.in_proj_bias.grad.clone()
        pre.step()
        torch.cuda.synchronize()
        w = model.layer.self_attn.in_proj_weight.grad
        assert torch.equal(w[64:128], raw[64:128]) and torch.equal(model.layer.self_attn.in_proj_bias.grad[64:128],
                                                                   rawb[64:128])
        assert not torch.equal(w[:64], raw[:64])


def _run_dist(backend):
    import os
    import socket
    import subprocess
    import sys
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    port = s.getsockname()[1]
    s.close()
    script = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'dist_attention.py')
    out = subprocess.run([sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node=2',
                          '--master-addr', '127.0.0.1', '--master-port', str(port), script, '--backend', backend],
                         capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, (out.stdout[-3000:], out.stderr[-3000:])
    assert out.stdout.count('dist_attention ok') == 2, out.stdout[-2000:]


def test_two_ranks_gloo():
    _run_dist('gloo')


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason='NCCL needs one GPU per rank')
def test_two_ranks_nccl():
    _run_dist('nccl')


class LM(nn.Module):
    """The reference language-model example's shape: embedding, sequence-first encoder, untied decoder."""

    def __init__(self, V=500, E=64):
        super().__init__()
        self.encoder = nn.Embedding(V, E)
        layer = nn.TransformerEncoderLayer(E, 4, 128, dropout=0.1)
        self.transformer_encoder = nn.TransformerEncoder(layer, 2, enable_nested_tensor=False)
        self.decoder = nn.Linear(E, V)

    def forward(self, idx, mask):
        return self.decoder(self.transformer_encoder(self.encoder(idx), mask))


def test_language_model_example_trains():
    from kfac_b200.preconditioner import KFACPreconditioner
    torch.manual_seed(0)
    model = LM().to(DEV)
    pre = KFACPreconditioner(model, skip_layers=[], precondition_embeddings=True, diagonal_g_layers=['decoder'],
                             precondition_attention=True, damping=0.003)
    names = [n for n, _ in pre._layers.values()]
    assert sum(n.endswith(('q_proj', 'k_proj', 'v_proj', 'out_proj')) for n in names) == 8
    opt = torch.optim.SGD(model.parameters(), lr=0.1)
    idx = torch.randint(0, 500, (35, 8), device=DEV)
    mask = nn.Transformer.generate_square_subsequent_mask(34, device=DEV)
    losses = []
    for _ in range(8):
        opt.zero_grad()
        loss = F.cross_entropy(model(idx[:-1], mask).reshape(-1, 500), idx[1:].reshape(-1))
        loss.backward()
        pre.step()
        opt.step()
        losses.append(float(loss))
    assert all(v == v for v in losses) and losses[-1] < losses[0], losses
