"""Public drop-in class: `KFACPreconditioner(model, **kw).step()`.

Constructor signature, validation order, error messages and derived attributes
follow kfac/preconditioner.py:54-334 so a user of the reference can switch the
import and keep their training script:

    from kfac_b200.preconditioner import KFACPreconditioner
    preconditioner = KFACPreconditioner(model, ...)
    loss.backward(); preconditioner.step(); optimizer.step()
"""
from __future__ import annotations

import logging
import warnings
from typing import Any, Callable

import torch
import torch.distributed as dist

from kfac_b200 import attention, recurrent
from kfac_b200.assignment import KAISAAssignment
from kfac_b200.base_preconditioner import BaseKFACPreconditioner
from kfac_b200.distributed import ArenaCommunicator, get_rank, get_world_size
from kfac_b200.enums import (AllreduceMethod, AssignmentStrategy, ComputeMethod,
                             DistributedStrategy)
from kfac_b200.layers import KFACLayer, register_modules

logger = logging.getLogger(__name__)


def _mock_new_group(x: list[int]) -> None:
    return None


def layer_work(layers: dict[torch.nn.Module, tuple[str, KFACLayer]],
               assignment_strategy: AssignmentStrategy) -> dict[str, dict[str, float]]:
    """Per-factor cost the KAISA placement balances: d^3 (COMPUTE) or d^2 (MEMORY) for a dense factor.  A diagonal
    factor (an embedding's or a diagonal-A layer's A, a diagonal-G layer's G) is never decomposed and takes V floats, so its cost is V under
    both strategies; a V^3 cost would let one vocabulary dominate the greedy placement.  A tied pair is one unit
    under the embedding's name with the single factor 'G' (one rank holds E, H, f and h whatever colocate_factors
    says), costed 2 cost(d) + 2 V; the head has no entry."""
    if assignment_strategy == AssignmentStrategy.COMPUTE:
        cost = lambda n: n ** 3  # noqa: E731
    elif assignment_strategy == AssignmentStrategy.MEMORY:
        cost = lambda n: n ** 2  # noqa: E731
    else:
        raise AssertionError(f'Unknown assignment_strategy={assignment_strategy}')
    work = {}
    for name, l in layers.values():
        if l.tied_embedding is not None:
            continue
        if l.tied_head is not None:
            work[name] = {'G': 2 * cost(l.g_dim) + 2 * l.a_dim}
        else:
            work[name] = {'A': l.a_dim if l.diag_a else cost(l.a_dim), 'G': l.g_dim if l.diag_g else cost(l.g_dim)}
    return work


def _check_diagonal_layers(layers: dict[torch.nn.Module, tuple[str, KFACLayer]],
                           compute_method: ComputeMethod, tied_embeddings: bool = False) -> None:
    """Reject the registered diagonal layers (embeddings, diagonal-A and diagonal-G layers) this preconditioner cannot
    handle.  With
    `tied_embeddings`, an embedding whose weight is the weight of one bias-less diagonal-G Linear forms a tied pair
    with it instead (`KFACLayer.tied_head` / `tied_embedding`)."""
    diag = [(module, name, l) for module, (name, l) in layers.items() if l.diag_side]
    if tied_embeddings:
        _tie_pairs(layers, compute_method)
    for module, name, l in diag:
        bag = isinstance(module, torch.nn.EmbeddingBag)
        kind, keyword = (('embedding bag', 'precondition_embedding_bags') if bag
                         else ('embedding', 'precondition_embeddings') if l.embedding
                         else ('layer', 'diagonal_a_layers') if l.diag_a else ('layer', 'diagonal_g_layers'))
        if compute_method == ComputeMethod.EKFAC:
            raise ValueError(f'{keyword} does not support compute_method=EKFAC ({kind} "{name}"); '
                             f'add the {kind}s to skip_layers')
        if bag and module.mode == 'max':
            raise ValueError(f'embedding bag "{name}" has mode=\'max\': each output column reads a different row, so '
                             'it is not a Kronecker-factored layer (add it to skip_layers)')
        if l.embedding and module.sparse:
            raise ValueError(f'{kind} "{name}" has sparse=True: K-FAC needs a dense weight gradient '
                             '(add it to skip_layers or use sparse=False)')
        if l.embedding and module.scale_grad_by_freq:
            raise ValueError(f'{kind} "{name}" has scale_grad_by_freq=True: its weight gradient is then not the '
                             'one the K-FAC factors model (add it to skip_layers)')
        for other, (other_name, _) in layers.items():
            if l.tied_head is not None or l.tied_embedding is not None:
                break
            if other is not module and any(p is module.weight for p in other.parameters()):
                raise ValueError(f'{kind} "{name}" shares its weight with "{other_name}": two layers would '
                                 f'precondition one gradient; add one of them to skip_layers')


def _tie_pairs(layers: dict[torch.nn.Module, tuple[str, KFACLayer]], compute_method: ComputeMethod) -> None:
    """Form the tied pairs of precondition_tied_embeddings: a registered embedding and the one other registered module
    that owns its weight, which must be a bias-less torch.nn.Linear matched by diagonal_g_layers."""
    for module, (name, l) in layers.items():
        if not l.embedding or isinstance(module, torch.nn.EmbeddingBag):    # a bag never forms a pair
            continue
        owners = [(other, other_name, ol) for other, (other_name, ol) in layers.items()
                  if other is not module and any(p is module.weight for p in other.parameters())]
        if not owners:
            continue
        if len(owners) > 1:
            names = ', '.join(f'"{n}"' for _, n, _ in owners)
            raise ValueError(f'embedding "{name}" shares its weight with {names}: precondition_tied_embeddings pairs '
                             'one embedding with one head; add all but one of them to skip_layers')
        head, head_name, hl = owners[0]
        if not isinstance(head, torch.nn.Linear) or head.weight is not module.weight:
            raise ValueError(f'embedding "{name}" shares a weight with "{head_name}", which is not a torch.nn.Linear '
                             'using it as its weight: precondition_tied_embeddings ties an embedding to a Linear head '
                             'only; add one of them to skip_layers')
        if not hl.diag_g:
            raise ValueError(f'embedding "{name}" is tied to "{head_name}", which is not in diagonal_g_layers: '
                             f'precondition_tied_embeddings needs the head\'s diagonal G; add "{head_name}" to '
                             'diagonal_g_layers (or one of the two layers to skip_layers)')
        if head.bias is not None:
            raise ValueError(f'embedding "{name}" is tied to "{head_name}", which has a bias: '
                             'precondition_tied_embeddings supports bias-less heads only; add one of the two layers '
                             'to skip_layers')
        if compute_method == ComputeMethod.EKFAC:
            raise ValueError(f'precondition_tied_embeddings does not support compute_method=EKFAC (pair "{name}" / '
                             f'"{head_name}"); add one of the two layers to skip_layers')
        l.tied_head, hl.tied_embedding = hl, l
    # a weight shared by two Linears (with or without an embedding) stays refused by the checks that follow


def _enable_pi_damping(layers: dict[torch.nn.Module, tuple[str, KFACLayer]], compute_method: ComputeMethod) -> None:
    """Turn on pi-adjusted damping for every registered layer of the work assignment (normalization layers keep their
    damping), refusing the layers it does not cover."""
    for name, l in layers.values():
        if compute_method == ComputeMethod.EKFAC:
            raise ValueError(f'pi_damping does not support compute_method=EKFAC (layer "{name}"), which damps its '
                             'measured second moments directly; add the layers to skip_layers or set pi_damping=False')
        if l.tied_head is not None:
            head = next(n for n, hl in layers.values() if hl is l.tied_head)
            raise ValueError(f'pi_damping does not support the tied embedding / head pair "{name}" / "{head}"; add one '
                             'of the two layers to skip_layers or set pi_damping=False')
    for _, l in layers.values():
        l.pi_damping = True


class KFACPreconditioner(BaseKFACPreconditioner):
    """K-FAC gradient preconditioner with KAISA placement on H100 (sm_90a).

    `compute_method` takes EIGEN and INVERSE like the reference, and EKFAC: the eigen method with the
    Kronecker product of the eigenvalues replaced by second moments measured in the eigenbasis at every
    factor step (George et al., 2018).  EKFAC needs `grad_worker_fraction` to resolve to COMM_OPT,
    `accumulation_steps=1` and, for integer schedules, `inv_update_steps` a multiple of
    `factor_update_steps`; `compute_eigenvalue_outer_product` is ignored with it.

    `precondition_embeddings=True` also registers leaf `torch.nn.Embedding` modules (`EmbeddingBag` has its own
    keyword, `precondition_embedding_bags`), which
    the reference leaves to the first-order optimizer.  Their A factor is diagonal (the token frequencies) and
    kept as a vector; see `kfac_b200.layers.EmbeddingModuleHelper`.  The embedding's P is always formed from the
    eigenvalue vectors (`compute_eigenvalue_outer_product` does not apply to it, so no V x d matrix is stored),
    and its damping is the one of the step that preconditions.  It cannot be combined with EKFAC, sparse
    gradients, `scale_grad_by_freq`, or a weight shared with another registered module (a tied LM head; see
    `precondition_tied_embeddings`).

    `diagonal_g_layers` takes regexes matched against module names and class names, like `skip_layers`.  A
    registered `torch.nn.Linear` that matches keeps its G factor as the vector diag(G) of `out_features` floats
    (another registered module type that matches is an error; patterns that match nothing are not).  This is for
    layers with more outputs than the eigensolver takes (`KFAC_EIGH_MAX_N` = 8192), such as an untied LM head:
    A stays dense, and the layer's P is
        eigen:   P = [(grad Qa) / (dg x da + damping)] Qa^T
        inverse: P = diag(1 / (dg + damping)) grad (A + damping I)^-1
    with dg = diag(G) its own eigenvalues (Qg = I).  It is a different approximation of the curvature, not a faster
    path to the same one, hence opt-in.  `compute_eigenvalue_outer_product` does not apply to such a layer (no
    V x a matrix is stored) and its damping is the one of the step that preconditions.  It cannot be combined
    with EKFAC or with a weight shared with another registered module.

    `precondition_norms=True` also registers leaf `torch.nn.BatchNorm1d`, `BatchNorm2d`, `LayerNorm` and `RMSNorm`
    modules whose affine parameters require grad.  Their affine part y = s * xhat + b makes every channel c a one-input
    layer with bias on the normalized input, and its exact 2 x 2 Fisher block (1 x 1 without a bias) is kept instead
    of a Kronecker factorization:
        F_c = (1/N) sum_r g_rc^2 (xhat_rc, 1)(xhat_rc, 1)^T,    P_c = (F_c + damping I)^-1 (dW_c, db_c)
    with the rows of a Conv2d layer (scaled by 1/S) for BatchNorm on maps and sequences, and the rows of a Linear
    layer otherwise; see `kfac_b200.layers.NormModuleHelper`.  The blocks follow the factor schedule (EMA,
    `accumulation_steps`, the guarded EMA under a `grad_scaler`) and are snapshotted at inverse steps; P uses the
    damping of the step that preconditions and is the same under every `compute_method`.  Normalization layers take
    no part in the KAISA placement: every rank preconditions them locally from the all-reduced blocks.  Without
    SyncBatchNorm the BatchNorm statistics are those of each rank's batch, so the all-reduced block is the mean of
    the ranks' blocks.  At factor steps each norm call's input is held until its output's gradient arrives; inside a
    non-reentrant `torch.utils.checkpoint` region that keeps activations the checkpointing would drop.  Not
    registered: modules without affine parameters, SyncBatchNorm, BatchNorm3d, and GroupNorm and InstanceNorm*, which
    `precondition_group_norms` covers.

    `precondition_group_norms=True` also registers leaf `torch.nn.GroupNorm`, `InstanceNorm1d`, `InstanceNorm2d` and
    `InstanceNorm3d` modules whose affine parameters exist and all require grad: the normalization of diffusion U-Nets
    (`GroupNorm(32, C)`), ConvNeXt-style `GroupNorm(1, C)`, and image-to-image and 3-D medical generators
    (`InstanceNorm2d/3d(affine=True)`).  They take the blocks, P, schedule and local handling of `precondition_norms`
    with xhat normalized per example and group: for input (B, C, *) with S = prod(*) positions and G groups of
    Cg = C / G channels (G = C for an InstanceNorm), mu and the biased variance are those of the Cg * S entries of
    each example's group, and the rows are BatchNorm's (N = B * S positions, a_r and g_r scaled by 1/S; S = 1 for a
    GroupNorm on (B, C)).  An unbatched InstanceNorm input is one example.  The statistics are exact per example, so
    with several ranks the all-reduced block is the mean of the ranks' blocks.  The keyword is independent of
    `precondition_norms`; both may be on.  Not registered: modules without affine parameters or with a frozen one.
    A `diagonal_g_layers` match is a ValueError, and `skip_layers` takes precedence.

    `kfac_approx` chooses the statistics of weight-sharing layers (Eschenhagen et al., 2023): a `torch.nn.Linear`
    on (B, ..., d) applies one weight at R = numel / (B * d) positions of each example, a `torch.nn.Conv2d` at
    R = Ho * Wo.  'expand' (the default, the reference's) makes every position a row.  'reduce' makes every example
    one row, formed from the expand rows:
        x_b = (1/R) sum_t x_bt,    g_b = R^-1/2 sum_t g_bt,    A = (1/B) sum_b x_b x_b^T,    G = (1/B) sum_b g_b g_b^T
    (the conv rows keep their 1/Ho*Wo scaling, the ones column is averaged with the others).  It is a different
    approximation, R times cheaper to form: A is unchanged when x is constant over the positions and E[G] is unchanged
    when g is uncorrelated over them, so `damping` and `kl_clip` keep their scale.  It applies to dense and
    diagonal-G Linear layers and to Conv2d layers; a call with R = 1 (a Linear on (B, d), a conv with a 1 x 1 output)
    takes the expand path with the same bits.  Dimension 0 is always the example dimension: a sequence-first input
    (T, B, d) is read as T examples.  Embeddings (their diagonal A counts one-hot rows) and normalization layers (their
    exact per-channel blocks) keep their statistics.  Under EKFAC the reduced rows are the rows of S_batch (N = B),
    which makes it the per-example EKFAC of George et al.  Factor shapes do not change, so checkpoints move between the
    two settings.

    `precondition_attention=True` registers every `torch.nn.MultiheadAttention` whose parameters all require grad, and
    which `skip_layers` does not match by name or class, as four K-FAC layers `{name}.q_proj`, `.k_proj`, `.v_proj`
    and `.out_proj`, each preconditioned exactly like the `torch.nn.Linear` it is mathematically (rows [0, E), [E, 2E)
    and [2E, 3E) of `in_proj_weight` / `in_proj_bias` or the separate `q/k/v_proj_weight`, and `out_proj`); see
    `kfac_b200.layers.AttentionProjectionHelper`.  A `skip_layers` pattern matching one projection name leaves that
    projection's rows of the gradient untouched.  The `out_proj` leaf of an attention is never registered as a Linear
    (torch's attention never calls its forward, so its hooks could not fire).  To see the projections, the constructor
    sets the class of each registered attention to `kfac_b200.attention.KFACMultiheadAttention`, a subclass that adds
    no state and overrides only `forward`: at the factor steps in training it runs a restatement of torch's training
    path with the taps, and the stock forward otherwise.  Under `kfac_approx='reduce'` the example dimension is the
    attention's batch dimension (an unbatched call is one example).  Refused with a ValueError: `add_bias_kv`,
    `add_zero_attn`, subclasses of `torch.nn.MultiheadAttention`, a `diagonal_g_layers` pattern matching an attention or
    a projection, and a projection weight shared with another registered module.

    `precondition_tied_embeddings=True` preconditions a weight tied between a registered embedding
    (`precondition_embeddings`) and a bias-less `torch.nn.Linear` head in `diagonal_g_layers` (GPT-2, nanoGPT), instead
    of refusing it.  Both uses keep their statistics: the embedding's token frequencies f and G factor E, the head's A
    factor H and diagonal G h.  With the uses treated as uncorrelated and the factor-wise damping t of the inverse
    step, row v of the (V, d) gradient is preconditioned by
        F_v = (f_v + t)(E + t I) + (h_v + t)(H + t I),    P_v = F_v^-1 grad_v,
    solved exactly for all rows through the simultaneous diagonalisation M^T (E + t I) M = I,
    M^T (H + t I) M = diag(mu):  P = [(grad M) / ((f + t) 1^T + (h + t) mu^T)] M^T.  The pair is one unit of the
    placement (one rank decomposes E and the whitened H), P is stored and written back once, under every
    compute_method; `state_dict()` keeps both members' entries with their untied shapes.  Refused with a ValueError:
    a tied head outside `diagonal_g_layers`, a tied head with a bias, a weight owned by more than two registered
    modules or by two Linears, and EKFAC.  With `skip_layers` matching either member there is no pair.

    `precondition_conv_nd=True` also registers leaf `torch.nn.Conv1d` and `torch.nn.Conv3d` modules whose parameters
    all require grad (audio and sequence encoders, TCNs, video and volumetric models), which the reference leaves to
    the first-order optimizer.  Their statistics are those of a Conv2d layer on the N-d lattice (rows = B * S positions,
    S = Lo or Do * Ho * Wo, A and G rows scaled by 1/S; A's features in the order (C_in, kd, kh, kw) [+ ones] of
    `weight.reshape(out, -1)`), but unlike Conv2d the geometry is honoured exactly: dilation on every axis, integer,
    'valid' or 'same' padding (asymmetric where torch pads so), and a `padding_mode` other than 'zeros' by padding the
    input as the module's forward does.  An unbatched input is one example.  A Conv1d with dilation 1 and zero padding
    has the factors of its Conv2d twin with kernel (1, k) on the unsqueezed input.  It works with `kfac_approx`
    ('reduce': R = S), EKFAC, `grad_scaler`, `accumulation_steps` and `factor_dtype`; see
    `kfac_b200.layers.ConvNdModuleHelper`.  Refused with a ValueError naming the layer: `groups != 1`, an A dimension
    C_in * kd * kh * kw (+ bias) or `out_channels` above `KFAC_EIGH_MAX_N` (8192), and a `diagonal_g_layers` match.
    Conv2d layers are unaffected by the keyword.

    `precondition_conv_transpose=True` also registers leaf `torch.nn.ConvTranspose1d`, `ConvTranspose2d` and
    `ConvTranspose3d` modules whose parameters all require grad: the upsampling layers of DCGAN-style generators, U-Net
    and FCN decoders, 1-D audio upsamplers and 3-D segmentation decoders, which the reference leaves to the first-order
    optimizer.  Output position o of such a layer reads input (o + p - k d) / s through tap k where s divides
    (o + p - k d), zero elsewhere; its rows are the B * S output positions with the Conv2d constants (A and G rows
    scaled by 1/S, 'reduce': R = S), A's features (C_in, kd, kh, kw) [+ ones] and G C_out x C_out.  The gradient
    matrix is the weight gradient (C_in, C_out, k...) permuted to (C_out, C_in * K); the precondition, the kl-clip
    inner product and the write-back read and write the weight gradient in place in its own layout.  `output_size`,
    positional or keyword, sets the output padding as the module's forward does.  It works with unbatched inputs,
    `kfac_approx`, EKFAC, `grad_scaler`, `accumulation_steps`, `factor_dtype` and every distributed strategy; see
    `kfac_b200.layers.ConvTransposeModuleHelper`.  Refused with a ValueError naming the layer and `skip_layers`:
    `groups != 1`, an A dimension C_in * K (+ bias) or `out_channels` above `KFAC_EIGH_MAX_N` (8192), more than 2048
    taps under 'reduce', and a `diagonal_g_layers` match.

    `precondition_recurrent=True` registers every `torch.nn.RNN` (tanh and relu), `torch.nn.LSTM` and `torch.nn.GRU`
    whose parameters all require grad, and which `skip_layers` does not match by name or class, as two K-FAC layers per
    layer k and direction (sfx '' or '_reverse'): `{name}.ih_l{k}{sfx}` (`weight_ih` / `bias_ih`; A: the layer input,
    G: the gradient of the input projection) and `{name}.hh_l{k}{sfx}` (`weight_hh` / `bias_hh`; A: the previous hidden
    state h_{t-1} of that direction, h0 at the first position, zeros when `hx` is not passed; G: the gradient of the
    hidden projection, equal to the input one for RNN and LSTM and [dr, dz, r * dn] for GRU).  Time steps are the
    positions of a weight-shared Linear layer (the "independent time steps" model of Martens, Ba & Johnson, 2018):
    N = T * B positions, or the sum of the lengths of a PackedSequence, with A and G scaled by 1/N; under
    `kfac_approx='reduce'` each sequence is one example (R_b = T or its length).  For RNN and LSTM, `bias_ih` and
    `bias_hh` have the same gradient; each is preconditioned by its own layer with its own ones column, as in the
    two-`nn.Linear` twin of the module.  Placement, collectives, `state_dict()` and `memory_usage()` are those of that
    twin.  A `skip_layers` pattern matching one sub-layer name leaves that sub-layer's gradients untouched.  To see the
    projections, the constructor sets the class of each registered module to `kfac_b200.recurrent.KFACRNN`, `KFACLSTM`
    or `KFACGRU`, subclasses that add no state and override only `forward`: at the factor steps in training it runs a
    restatement of torch's forward with a time loop (its inter-layer dropout mask is drawn differently from cuDNN's),
    and the stock forward (cuDNN) otherwise.  Refused with a ValueError naming the layer and `skip_layers`:
    `proj_size > 0`, a factor above `KFAC_EIGH_MAX_N` (8192; an LSTM with H > 2048, a GRU with H > 2730), a
    `diagonal_g_layers` match, a weight shared with another registered module, and subclasses.

    `diagonal_a_layers` takes regexes matched against module names and class names, like `diagonal_g_layers`.  A
    registered `torch.nn.Linear` or `torch.nn.Conv2d` (and, with `precondition_conv_nd`, `Conv1d` / `Conv3d`) that
    matches keeps its A factor as the vector diag(A) of `a_dim` floats, bias entry included: the diagonal of the dense A
    the layer would form from the same rows (the conv rows' 1/S, the K-FAC-reduce rows), with the same EMA,
    `accumulation_steps`, schedules and `grad_scaler` handling.  This is for layers with more inputs than the
    eigensolver takes (`KFAC_EIGH_MAX_N` = 8192): the `down_proj` of a LLaMA-style MLP (11008 or 14336 inputs), or a
    3 x 3 convolution on 1024 or 1280 channels (A = 9217 or 11521).  G stays dense (and must be at most 8192), and the
    layer's P is
        eigen:   P = Qg [(Qg^T grad) / (dg x da + damping)]
        inverse: P = (G + damping I)^-1 grad diag(1 / (da + damping))
    with da = diag(A) its own eigenvalues (Qa = I).  It is a different approximation of the curvature, hence opt-in.
    As for diagonal-G layers, `compute_eigenvalue_outer_product` does not apply and the damping is the one of the step
    that preconditions; P keeps the dense layout, so kl-clip and the write-back are unchanged.  Refused with a
    ValueError naming the layer and `skip_layers`: EKFAC, a match on an embedding, a normalization layer, an attention
    projection, a recurrent sub-layer or a transposed convolution, a layer matched by `diagonal_g_layers` too, a G
    above 8192, and a weight shared with another registered module.

    `pi_damping=True` splits the damping between the two Kronecker factors of every registered layer by their trace
    norms (factored Tikhonov damping with the trace-norm pi, Martens & Grosse 2015, sec. 6.3; `compute_pi_tracenorm` in
    TF K-FAC, pi-adjusted damping in KFAC-JAX).  A (x) G equals cA (x) G/c for any c > 0, and how a layer's statistics
    split the scale between A and G differs a lot between layer kinds (a conv layer's 1/S, an embedding's token
    frequencies, a loss that is a mean over tokens).  With
        pi = sqrt((tr A / a_dim) / (tr G / g_dim)),    s = sqrt(damping),    gamma_A = s pi,    gamma_G = s / pi
    (pi = 1 where a mean trace is not a positive finite number; a diagonal factor's trace is the sum of its vector) the
    layer is preconditioned by (A + gamma_A I) (x) (G + gamma_G I), which does not depend on that split:
        eigen:   P = Qg [(Qg^T grad Qa) / ((dg + gamma_G) x (da + gamma_A))] Qa^T
        inverse: P = (G + gamma_G I)^-1 grad (A + gamma_A I)^-1
    and the same formulas for embeddings, diagonal-G and diagonal-A layers.  This is the Tikhonov damping of the
    product, so each factor receives sqrt(damping): the inverse method's damping changes meaning relative to
    `pi_damping=False`.  pi is formed at every inverse step (and by `load_state_dict(compute_inverses=True)`) from the
    factors that step decomposes, by every rank for every layer, and kept until the next inverse step; it needs no
    collective and is not part of `state_dict()`.  The damping of the inverse step forms dgda and the inverses, the
    damping of the step that preconditions divides by the eigenvalues without `compute_eigenvalue_outer_product` and
    by the diagonal factors.  Normalization layers keep their blocks damped by `damping`.  Refused with a ValueError
    naming the layer: EKFAC (which damps its measured S directly) and tied embedding / head pairs.

    `precondition_embedding_bags=True` also registers leaf `torch.nn.EmbeddingBag` modules whose weight requires grad
    (the bag-of-tokens text classifier, fastText-style n-gram models, the sparse-feature tables of DLRM-style
    recommenders), independently of `precondition_embeddings`.  A call of B bags is a Linear layer on the pooled rows
    c_b in R^V (c_bv the sum of the `per_sample_weights`, or 1, of bag b's entries equal to v for mode='sum'; their
    count over the bag's non-padding entries for mode='mean'; `padding_idx` entries left out), so its A factor
    (1/B) C^T C is V x V.  The bag keeps its diagonal A_v = (1/B) sum_b c_bv^2, a vector of V floats, exact for bags
    of one index (where it is `nn.Embedding`'s A); this is a different approximation from the exact Fisher, hence
    opt-in.  Every bag, empty or not, is one row, also under `kfac_approx='reduce'`.  G comes from the (B, d) output
    gradient, and P, placement, collectives, `state_dict()` (A as a V-vector) and `memory_usage()` are an embedding's.
    1-D indices with `offsets` (with or without `include_last_offset`) and 2-D indices are supported.  Under a
    `grad_scaler` the bag's A takes the guarded EMA like a dense A (per-sample weights are forward values); without
    one, a non-finite A makes the next `step()` raise.  Refused with a ValueError naming the layer and `skip_layers`:
    mode='max', `sparse=True`, `scale_grad_by_freq=True`, EKFAC, a `diagonal_g_layers` or `diagonal_a_layers` match
    and a weight shared with another registered module.
    """

    def __init__(
        self,
        model: torch.nn.Module,
        *,
        factor_update_steps: Callable[[int], int] | int = 1,
        inv_update_steps: Callable[[int], int] | int = 1,
        damping: Callable[[int], float] | float = 0.001,
        factor_decay: Callable[[int], float] | float = 0.95,
        kl_clip: Callable[[int], float] | float = 0.001,
        lr: Callable[[int], float] | float = 0.1,
        accumulation_steps: int = 1,
        allreduce_bucket_cap_mb: float = 25.0,
        assignment_strategy: AssignmentStrategy | str = AssignmentStrategy.COMPUTE,
        colocate_factors: bool = True,
        compute_method: ComputeMethod | str = ComputeMethod.EIGEN,
        compute_eigenvalue_outer_product: bool = True,
        grad_worker_fraction: DistributedStrategy | float = DistributedStrategy.COMM_OPT,
        symmetry_aware: bool = False,
        grad_scaler: Any | Callable[[], float] | None = None,
        factor_dtype: torch.dtype | None = None,
        inv_dtype: torch.dtype = torch.float32,
        skip_layers: list[str] | None = None,
        update_factors_in_hook: bool = True,
        loglevel: int = logging.DEBUG,
        precondition_embeddings: bool = False,
        diagonal_g_layers: list[str] | None = None,
        precondition_norms: bool = False,
        kfac_approx: str = 'expand',
        precondition_attention: bool = False,
        precondition_tied_embeddings: bool = False,
        precondition_conv_nd: bool = False,
        precondition_conv_transpose: bool = False,
        precondition_group_norms: bool = False,
        precondition_recurrent: bool = False,
        diagonal_a_layers: list[str] | None = None,
        pi_damping: bool = False,
        precondition_embedding_bags: bool = False,
    ) -> None:
        if not isinstance(pi_damping, bool):
            raise ValueError(f'pi_damping must be a bool, got {pi_damping!r}')
        if allreduce_bucket_cap_mb < 0:
            raise ValueError('allreduce_bucket_cap_mb must be >= 0')
        if kfac_approx not in ('expand', 'reduce'):
            raise ValueError(f"kfac_approx must be 'expand' or 'reduce', got {kfac_approx!r}")
        if isinstance(assignment_strategy, str):
            assignment_strategy = AssignmentStrategy[assignment_strategy.upper()]
        if isinstance(compute_method, str):
            compute_method = ComputeMethod[compute_method.upper()]
        if (compute_method == ComputeMethod.EIGEN and compute_eigenvalue_outer_product
                and not colocate_factors):
            raise ValueError('colocate_factors must be True to use compute_eigenvalue_outer_product')
        # factors and second-order data are STORED in float32 arenas (tensor-core 3xTF32 with fp32
        # accumulation has no fp64 path): float64 is accepted and cast at the boundary, half-precision
        # factor dtypes round the hook inputs like the reference does (kfac/layers/base.py:350,364)
        if factor_dtype not in (None, torch.float32, torch.float64, torch.float16, torch.bfloat16):
            raise ValueError(f'unsupported factor_dtype {factor_dtype}')
        if inv_dtype not in (torch.float32, torch.float64):
            raise ValueError(
                'kfac_b200 computes the eigendecompositions and the precondition in float32 (like '
                'kfac/layers/eigen.py:310-312); inv_dtype must be float32 or float64 (cast at the boundary), '
                f'got {inv_dtype}')

        size = get_world_size()
        if isinstance(grad_worker_fraction, DistributedStrategy):
            distributed_strategy = grad_worker_fraction
            if distributed_strategy == DistributedStrategy.COMM_OPT:
                grad_worker_fraction = 1.0
            elif distributed_strategy == DistributedStrategy.HYBRID_OPT:
                grad_worker_fraction = 0.5
            elif distributed_strategy == DistributedStrategy.MEM_OPT:
                grad_worker_fraction = 1.0 / size
            else:
                raise AssertionError(f'Unknown enum {grad_worker_fraction}')
        else:
            if not 0 <= grad_worker_fraction or not 1 >= grad_worker_fraction:
                raise ValueError('grad_worker_fraction must in [0, 1]')
            if grad_worker_fraction == 0:
                grad_worker_fraction = 1.0 / size
            if size % max(1, round(size * grad_worker_fraction)) != 0:
                raise ValueError('grad_worker_fraction must produce groups of equal size')
            if grad_worker_fraction == 1:
                grad_worker_fraction = 1.0
                distributed_strategy = DistributedStrategy.COMM_OPT
            elif grad_worker_fraction <= 1 / size:
                distributed_strategy = DistributedStrategy.MEM_OPT
            else:
                distributed_strategy = DistributedStrategy.HYBRID_OPT
        assert isinstance(grad_worker_fraction, float)

        if compute_method == ComputeMethod.EKFAC:
            if distributed_strategy != DistributedStrategy.COMM_OPT:
                raise ValueError('compute_method=EKFAC needs grad_worker_fraction to resolve to COMM_OPT '
                                 '(every rank holds the eigenbases and measures its rows in them)')
            if accumulation_steps != 1:
                raise ValueError('compute_method=EKFAC needs accumulation_steps=1')
            if (not callable(inv_update_steps) and not callable(factor_update_steps) and factor_update_steps > 0
                    and inv_update_steps % factor_update_steps != 0):
                raise ValueError('compute_method=EKFAC needs inv_update_steps to be a multiple of factor_update_steps')

        if not colocate_factors and distributed_strategy is DistributedStrategy.MEM_OPT:
            warnings.warn('grad_worker_frac=1/world_size (MEM_OPT) requires '
                          'colocate_factors=True. Enabling colocate_factors.', stacklevel=2)
            colocate_factors = True

        self.allreduce_bucket_cap_mb = allreduce_bucket_cap_mb
        self.assignment_strategy = assignment_strategy
        self.colocate_factors = colocate_factors
        self.compute_eigenvalue_outer_product = compute_eigenvalue_outer_product
        self.compute_method = compute_method
        self.distributed_strategy = distributed_strategy
        self.grad_worker_fraction = grad_worker_fraction
        self.grad_scaler = grad_scaler
        self.factor_dtype = factor_dtype
        self.inv_dtype = inv_dtype
        self.skip_layers = [] if skip_layers is None else skip_layers
        self.symmetry_aware = symmetry_aware
        self.allreduce_method = (AllreduceMethod.ALLREDUCE_BUCKETED if allreduce_bucket_cap_mb > 0
                                 else AllreduceMethod.ALLREDUCE)
        self.tdc = ArenaCommunicator(bucket_cap_mb=allreduce_bucket_cap_mb)

        kfac_layers = register_modules(
            model, self.skip_layers, precondition_embeddings=precondition_embeddings,
            diagonal_g_layers=diagonal_g_layers, precondition_norms=precondition_norms, kfac_approx=kfac_approx,
            precondition_attention=precondition_attention, precondition_conv_nd=precondition_conv_nd,
            precondition_conv_transpose=precondition_conv_transpose,
            precondition_group_norms=precondition_group_norms,
            precondition_recurrent=precondition_recurrent, diagonal_a_layers=diagonal_a_layers,
            precondition_embedding_bags=precondition_embedding_bags, method=compute_method,
            prediv_eigenvalues=compute_eigenvalue_outer_product, grad_scaler=grad_scaler,
            factor_dtype=factor_dtype, inv_dtype=inv_dtype, symmetry_aware=symmetry_aware)
        # normalization layers are preconditioned locally on every rank: the placement never sees them
        norm_layers = {m: v for m, v in kfac_layers.items() if v[1].norm}
        kfac_layers = {m: v for m, v in kfac_layers.items() if not v[1].norm}
        _check_diagonal_layers(kfac_layers, compute_method, tied_embeddings=precondition_tied_embeddings)
        if pi_damping:
            _enable_pi_damping(kfac_layers, compute_method)
        for name, kfac_layer in list(kfac_layers.values()) + list(norm_layers.values()):
            logger.log(loglevel, f'Registered name="{name}": {repr(kfac_layer)}')

        work = layer_work(kfac_layers, assignment_strategy)

        assignment = KAISAAssignment(
            work, local_rank=get_rank(), world_size=size,
            grad_worker_fraction=grad_worker_fraction,
            group_func=dist.new_group if dist.is_initialized() else _mock_new_group,
            colocate_factors=colocate_factors)
        logger.log(loglevel, f'KFAC layer assignments: {assignment}')

        defaults = {
            'allreduce_bucket_cap_mb': allreduce_bucket_cap_mb,
            'allreduce_method': self.allreduce_method,
            'assignment_strategy': assignment_strategy,
            'colocate_factors': colocate_factors,
            'compute_eigenvalue_outer_product': compute_eigenvalue_outer_product,
            'compute_method': compute_method,
            'distributed_strategy': distributed_strategy,
            'grad_worker_fraction': grad_worker_fraction,
            'grad_scaler': grad_scaler is not None,
            'factor_dtype': factor_dtype,
            'inv_dtype': inv_dtype,
            'skip_layers': self.skip_layers,
            'symmetry_aware': symmetry_aware,
            'precondition_embeddings': precondition_embeddings,
            'diagonal_g_layers': diagonal_g_layers,
            'precondition_norms': precondition_norms,
            'kfac_approx': kfac_approx,
            'precondition_attention': precondition_attention,
            'precondition_tied_embeddings': precondition_tied_embeddings,
            'precondition_conv_nd': precondition_conv_nd,
            'precondition_conv_transpose': precondition_conv_transpose,
            'precondition_group_norms': precondition_group_norms,
            'precondition_recurrent': precondition_recurrent,
            'diagonal_a_layers': diagonal_a_layers,
            'pi_damping': pi_damping,
            'precondition_embedding_bags': precondition_embedding_bags,
        }
        super().__init__(
            kfac_layers, norm_layers=norm_layers, factor_update_steps=factor_update_steps,
            inv_update_steps=inv_update_steps, factor_decay=factor_decay, damping=damping,
            kl_clip=kl_clip, lr=lr, accumulation_steps=accumulation_steps,
            assignment=assignment, update_factors_in_hook=update_factors_in_hook,
            defaults=defaults, tdc=self.tdc, loglevel=loglevel)
        for module in self._attention_taps:
            attention.bind(module, self)
        for module in self._recurrent_taps:
            recurrent.bind(module, self)
