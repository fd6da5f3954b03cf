"""Wav2vec pre-training on the engine: the reference's ``Wav2Vec`` and ``ConstrastiveCriterion`` (rnnt/wav2vec.py),
``GumbelVectorQuantizer`` (modules/softmax_vector_quantizer.py) and the span mask (rnnt/data_utils.py:348-505).

Same constructors, defaults, submodule names, ``state_dict`` keys and seeded weights as the reference, so
cli/pretrain_wav2vec.py runs on the engine by importing these two classes from here.  The front end, the encoder and
every Linear run the engine's kernels (``set_precision`` / autocast select fp32 or bf16 mode); the span mask, the row
gathers, the quantizer, the contrastive logits and the cross-entropy run csrc/w2v.cu, deterministically.  The
quantizer statistics, the logits and the loss are fp32 in both modes.

Host-side random draws use the reference's generators in the reference's order, so equal seeds draw equal spans
(numpy's global generator) and equal negatives (torch's CPU generator); the Gumbel noise is drawn on the device by
``gumbel_noise`` exactly as F.gumbel_softmax draws it.  Each draw reaches the device in one non-blocking copy from
pinned memory, and a criterion call reads back to the host once, for its logging values.

Options the reference cannot run, or that no caller uses and that would break the per-utterance structure of the
logits, raise ValueError before any device work (DESIGN.md section 8 lists them)."""
import numpy as np
import torch
from torch import nn

from .. import functional as Fn
from .models import Encoder, FrontEnd, ResLayerNormGRU, ResLayerNormLSTM, _lens_to_device, _precision, _set_precision
from .tokenizer import NUL


def gumbel_noise(logits):
    """The Gumbel noise of F.gumbel_softmax(logits): -log(Exp(1)) drawn on logits' device, shape and dtype."""
    return -torch.empty_like(logits).exponential_().log()


def buffered_arange(max):
    """rnnt/data_utils.py:499-505: arange(max) as int64."""
    return torch.arange(max)


def compute_mask_indices(shape, padding_mask, mask_prob, mask_length, mask_type="static", mask_other=0.0,
                         min_masks=0, no_overlap=False, min_space=0):
    """rnnt/data_utils.py:348-471 for padding_mask None and no_overlap False (the reference fails on the other two):
    a [B, T] bool mask with the same number of masked frames in every row, drawn from numpy's global generator in the
    reference's order."""
    if padding_mask is not None:
        raise ValueError("compute_mask_indices: padding masks are not supported")
    if no_overlap:
        raise ValueError("compute_mask_indices: no_overlap=True is not supported (the reference uses np.int)")
    bsz, all_sz = shape
    mask = np.full((bsz, all_sz), False)
    all_num_mask = int(mask_prob * all_sz / float(mask_length) + np.random.rand())
    all_num_mask = max(min_masks, all_num_mask)
    mask_idcs = []
    for _ in range(bsz):
        sz, num_mask = all_sz, all_num_mask
        if mask_type == "static":
            lengths = np.full(num_mask, mask_length)
        elif mask_type == "uniform":
            lengths = np.random.randint(mask_other, mask_length * 2 + 1, size=num_mask)
        elif mask_type == "normal":
            lengths = np.random.normal(mask_length, mask_other, size=num_mask)
            lengths = [max(1, int(round(x))) for x in lengths]
        elif mask_type == "poisson":
            lengths = np.random.poisson(mask_length, size=num_mask)
            lengths = [int(round(x)) for x in lengths]
        else:
            raise ValueError("unknown mask selection " + str(mask_type))
        if sum(lengths) == 0:
            lengths[0] = min(mask_length, sz - 1)
        min_len = min(lengths)
        if sz - min_len <= num_mask:
            min_len = sz - num_mask - 1
        mask_idc = np.random.choice(sz - min_len, num_mask, replace=False)
        mask_idc = np.asarray([mask_idc[j] + offset for j in range(len(mask_idc)) for offset in range(lengths[j])])
        mask_idcs.append(np.unique(mask_idc[mask_idc < sz]))
    min_len = min([len(m) for m in mask_idcs])
    for i, mask_idc in enumerate(mask_idcs):
        if len(mask_idc) > min_len:
            mask_idc = np.random.choice(mask_idc, min_len, replace=False)
        mask[i, mask_idc] = True
    return mask


def sample_negative_indices(B, M, K):
    """Wav2Vec.sample_negatives' draw (rnnt/wav2vec.py:205-261) as frame indices within each utterance: torch.randint on
    the CPU generator, bumped past the frame itself; negative k of masked frame m is entry [b, m*K + k]."""
    if M < 2:
        raise ValueError("sampling negatives needs at least 2 masked frames per utterance, got %d" % M)
    tszs = buffered_arange(M).unsqueeze(-1).expand(-1, K).flatten()
    neg = torch.randint(low=0, high=M - 1, size=(B, K * M))
    neg[neg >= tszs] += 1
    return neg


def _to_device_i32(a, device):
    return _lens_to_device(torch.from_numpy(np.ascontiguousarray(a, dtype=np.int32)), device)


def _check_bf16_linear(lin, name):
    if lin.in_features % 8 or lin.out_features % 8:
        raise ValueError("bf16 mode needs %s's widths to be multiples of 8 (got %d -> %d); use set_precision('fp32')"
                         % (name, lin.in_features, lin.out_features))


class GumbelVectorQuantizer(nn.Module):
    """modules/softmax_vector_quantizer.py:11-201, same constructor, parameters and seeded weights.  forward runs
    weight_proj through Fn.Linear and the rest through Fn.W2VQuantize; it implements combine_groups=False,
    time_first=True and weight_proj_depth=1, what Wav2Vec builds."""

    def __init__(self, dim, num_vars, temp, groups, combine_groups, vq_dim, time_first, activation=nn.GELU(),
                 weight_proj_depth=1, weight_proj_factor=1):
        super().__init__()
        self.groups = groups
        self.combine_groups = combine_groups
        self.input_dim = dim
        self.num_vars = num_vars
        self.time_first = time_first
        assert vq_dim % groups == 0, f"dim {vq_dim} must be divisible by groups {groups} for concatenation"
        var_dim = vq_dim // groups
        num_groups = groups if not combine_groups else 1
        self.vars = nn.Parameter(torch.FloatTensor(1, num_groups * num_vars, var_dim))
        nn.init.uniform_(self.vars)
        if weight_proj_depth > 1:
            def block(input_dim, output_dim):
                return nn.Sequential(nn.Linear(input_dim, output_dim), activation)
            inner_dim = self.input_dim * weight_proj_factor
            self.weight_proj = nn.Sequential(
                *[block(self.input_dim if i == 0 else inner_dim, inner_dim) for i in range(weight_proj_depth - 1)],
                nn.Linear(inner_dim, groups * num_vars))
        else:
            self.weight_proj = nn.Linear(self.input_dim, groups * num_vars)
            nn.init.normal_(self.weight_proj.weight, mean=0, std=1)
            nn.init.zeros_(self.weight_proj.bias)
        if isinstance(temp, str):
            import ast
            temp = ast.literal_eval(temp)
        assert len(temp) == 3, f"{temp}, {len(temp)}"
        self.max_temp, self.min_temp, self.temp_decay = temp
        self.curr_temp = self.max_temp
        self.codebook_indices = None

    def set_num_updates(self, num_updates):
        self.curr_temp = max(self.max_temp * self.temp_decay ** num_updates, self.min_temp)

    def _check(self):
        if self.combine_groups or not self.time_first or not isinstance(self.weight_proj, nn.Linear):
            raise ValueError("edgedict_b200 implements GumbelVectorQuantizer with combine_groups=False, time_first=True "
                             "and weight_proj_depth=1")
        if _precision(self) == "bf16":
            _check_bf16_linear(self.weight_proj, "weight_proj")

    def forward(self, x, produce_targets=False):
        """x [B, T, dim] -> the reference's dict: x [B, T, vq_dim], num_vars, code_perplexity, prob_perplexity, temp
        and, with produce_targets, targets [B, T, groups] (int64)."""
        self._check()
        bsz, tsz, fsz = x.shape
        G, V = self.groups, self.num_vars
        lin = self.weight_proj
        logits = Fn.Linear.apply(x.reshape(-1, fsz), lin.weight, lin.bias, _precision(self))
        noise = gumbel_noise(logits.view(-1, V)).view(logits.shape) if self.training else None
        q, pp, cp, k = Fn.W2VQuantize.apply(logits, self.vars, noise, G, float(self.curr_temp))
        result = {"num_vars": V * G, "code_perplexity": cp, "prob_perplexity": pp, "temp": self.curr_temp}
        if produce_targets:
            result["targets"] = k.view(bsz, tsz, G).long()
        result["x"] = q.view(bsz, tsz, -1)
        return result


class Wav2Vec(nn.Module):
    """rnnt/wav2vec.py:20-421: same constructor, defaults, submodules, ``state_dict`` keys and seeded weights.

    ``feature_grad_mult`` is accepted and ignored, as in the reference, whose forward never reads it.  ``layer_norm``
    is built (it consumes no generator state but is a checkpoint key) and, as in the reference, never used."""

    def __init__(self,
                 frontend_params=[(10, 5, 16)] + [(8, 4, 32)] + [(4, 2, 128)] * 3,
                 front_bias=False,
                 input_size=768,
                 enc_hidden_size=768, enc_layers=7, enc_dropout=0.1, enc_proj_size=512,
                 blank=NUL, module_type='LSTM', output_loss=True,
                 quantize_input=False,
                 quantize_targets=False,
                 same_quantizer=False,
                 mask_prob=0.15,
                 mask_length=10,
                 mask_selection='static',
                 mask_other=0.0,
                 mask_channel_prob=0.0,
                 mask_channel_selection='static',
                 mask_channel_other=0,
                 mask_channel_min_space=1,
                 no_mask_channel_overlap=False,
                 no_mask_overlap=False,
                 mask_min_space=1,
                 dropout_input=0.0,
                 dropout_features=0.0,
                 num_negatives=100,
                 negatives_from_everywhere=False,
                 cross_sample_negatives=0,
                 codebook_negatives=0,
                 final_dim=0,
                 latent_groups=2,
                 latent_dim=0,
                 target_glu=False,
                 latent_vars=320,
                 feature_grad_mult=1.0,
                 logit_temp=0.1,
                 latent_temp=(2, 0.5, 0.999995)):
        super().__init__()
        self.blank = blank
        self.quantize_input = quantize_input
        if module_type not in ['GRU', 'LSTM']:
            raise ValueError('Unsupported module type')
        module = ResLayerNormGRU if module_type == 'GRU' else ResLayerNormLSTM
        # the reference's creation order: every Linear and uniform_ below draws from the CPU generator
        self.encoder = Encoder(input_size=input_size, hidden_size=enc_hidden_size, num_layers=enc_layers,
                               dropout=enc_dropout, proj_size=enc_proj_size, module=module, time_reductions=[])
        self.frontend = FrontEnd(frontend_params, bias=front_bias)
        self.encoder_embed_dim = input_size
        self.embed = frontend_params[-1][-1]
        self.post_extract_proj = (nn.Linear(self.embed, input_size)
                                  if self.embed != input_size and not quantize_input else None)
        self.layer_norm = nn.LayerNorm(self.embed)
        self.mask_emb = nn.Parameter(torch.FloatTensor(self.encoder_embed_dim).uniform_())
        self.post_extract_proj = (nn.Linear(self.embed, self.encoder_embed_dim)
                                  if self.embed != self.encoder_embed_dim and not quantize_input else None)
        self.dropout_input = nn.Dropout(dropout_input)
        self.dropout_features = nn.Dropout(dropout_features)

        self.mask_prob = mask_prob
        self.mask_selection = mask_selection
        self.mask_channel_prob = mask_channel_prob
        self.mask_other = mask_other
        self.mask_length = mask_length
        self.no_mask_overlap = no_mask_overlap
        self.mask_min_space = mask_min_space

        self.quantizer = None
        self.input_quantizer = None
        self.n_negatives = num_negatives
        self.cross_sample_negatives = cross_sample_negatives
        self.codebook_negatives = codebook_negatives
        self.negatives_from_everywhere = negatives_from_everywhere
        self.logit_temp = logit_temp

        final_dim = final_dim if final_dim > 0 else self.encoder_embed_dim
        if quantize_targets:
            vq_dim = latent_dim if latent_dim > 0 else final_dim
            self.quantizer = GumbelVectorQuantizer(dim=self.embed, num_vars=latent_vars, temp=latent_temp,
                                                   groups=latent_groups, combine_groups=False, vq_dim=vq_dim,
                                                   time_first=True)
            self.project_q = nn.Linear(vq_dim, final_dim)
        else:
            self.project_q = nn.Linear(self.embed, final_dim)

        if quantize_input:
            if same_quantizer and self.quantizer is not None:
                vq_dim = final_dim
                self.input_quantizer = self.quantizer
            else:
                vq_dim = latent_dim if latent_dim > 0 else self.encoder_embed_dim
                self.input_quantizer = GumbelVectorQuantizer(dim=self.embed, num_vars=latent_vars, temp=latent_temp,
                                                             groups=latent_groups, combine_groups=False,
                                                             vq_dim=vq_dim, time_first=True)
            self.project_inp = nn.Linear(vq_dim, self.encoder_embed_dim)

        self.target_glu = None
        if target_glu:
            self.target_glu = nn.Sequential(nn.Linear(final_dim, final_dim * 2), nn.GLU())
        self.final_proj = nn.Linear(enc_proj_size, final_dim)

    def set_precision(self, precision):
        return _set_precision(self, precision)

    def _check(self, source, padding_mask, mask, features_only):
        """Every refusal, before any device work."""
        if padding_mask is not None:
            raise ValueError("padding_mask is not supported: the reference calls _get_feat_extract_output_lengths, "
                             "which it does not define")
        if self.mask_channel_prob > 0:
            raise ValueError("mask_channel_prob > 0 is not supported: the reference never sets mask_channel_length")
        if self.no_mask_overlap:
            raise ValueError("no_mask_overlap=True is not supported: the reference's compute_mask_indices uses np.int")
        if self.mask_selection not in ("static", "uniform", "normal", "poisson"):
            raise ValueError("unknown mask selection %r" % (self.mask_selection,))
        if not features_only:
            self._check_head(mask)
        if not isinstance(source, torch.Tensor) or not source.is_cuda or source.dtype != torch.float32:
            raise ValueError("Wav2Vec needs float32 CUDA audio (there is no CPU path)")

    def _check_head(self, mask):
        if not mask:
            raise ValueError("mask=False is supported with features_only=True only: the logits need masked frames")
        if not self.mask_prob > 0:
            raise ValueError("mask_prob must be > 0 unless features_only=True: the logits need masked frames")
        if self.negatives_from_everywhere:
            raise ValueError("negatives_from_everywhere=True is not supported: the reference unpacks the quantizer's "
                             "result dict")
        if not self.training and self.quantizer is None:
            raise ValueError("eval mode needs quantize_targets=True: the reference's targets come from its quantizer")
        if self.cross_sample_negatives > 0:
            raise ValueError("cross_sample_negatives > 0 is not supported")
        if self.codebook_negatives > 0:
            raise ValueError("codebook_negatives > 0 is not supported")
        if self.target_glu is not None:
            raise ValueError("target_glu=True is not supported")
        if self.n_negatives <= 0:
            raise ValueError("num_negatives must be > 0")
        if _precision(self) == "bf16":
            for name in ("post_extract_proj", "project_q", "project_inp", "final_proj"):
                lin = getattr(self, name, None)
                if lin is not None:
                    _check_bf16_linear(lin, name)
            for qz in (self.quantizer, self.input_quantizer):
                if qz is not None:
                    qz._check()

    def forward(self, source, padding_mask=None, mask=True, features_only=False):
        self._check(source, padding_mask, mask, features_only)
        if source.dim() == 3 and source.shape[1] == 1:
            source = source[:, 0]
        B, T = source.shape[0], self.frontend.output_length(source.shape[-1])
        dev = source.device
        p = _precision(self)

        idx = inv = neg = None
        if mask and self.mask_prob > 0:
            m = compute_mask_indices((B, T), None, self.mask_prob, self.mask_length, self.mask_selection,
                                     self.mask_other, min_masks=2, no_overlap=self.no_mask_overlap,
                                     min_space=self.mask_min_space)
            M = int(m[0].sum())
            frames = np.nonzero(m)[1].reshape(B, M)
            inv_h = np.full((B, T), -1, dtype=np.int32)
            inv_h[np.repeat(np.arange(B), M), frames.reshape(-1)] = np.tile(np.arange(M, dtype=np.int32), B)
            both = _to_device_i32(np.concatenate([frames.reshape(-1), inv_h.reshape(-1)]), dev)
            idx, inv = both[:B * M].view(B, M), both[B * M:].view(B, T)

        features = self.frontend(source)
        features_pen = Fn.W2VSqMean.apply(features)
        unmasked_features = features
        if self.post_extract_proj is not None:
            lin = self.post_extract_proj
            features = Fn.Linear.apply(features, lin.weight, lin.bias, p)
        features = self.dropout_input(features)
        unmasked_features = self.dropout_features(unmasked_features)

        num_vars = code_ppl = prob_ppl = curr_temp = None
        if self.input_quantizer:
            q = self.input_quantizer(features, produce_targets=False)
            num_vars, code_ppl, prob_ppl, curr_temp = q["num_vars"], q["code_perplexity"], q["prob_perplexity"], q["temp"]
            features = Fn.Linear.apply(q["x"], self.project_inp.weight, self.project_inp.bias, p)

        x = Fn.W2VMask.apply(features, self.mask_emb, idx, inv) if idx is not None else features
        x, _ = self.encoder(x)
        if features_only:
            return {"x": x, "padding_mask": padding_mask}

        y = Fn.W2VGather.apply(unmasked_features, idx, inv)
        M = idx.shape[1]
        result = {}
        if self.quantizer:
            q = self.quantizer(y, produce_targets=not self.training)
            num_vars, code_ppl, prob_ppl, curr_temp = q["num_vars"], q["code_perplexity"], q["prob_perplexity"], q["temp"]
            y = q["x"]
            if not self.training:
                result["targets"] = q["targets"]
        y = Fn.Linear.apply(y, self.project_q.weight, self.project_q.bias, p)
        neg = _to_device_i32(sample_negative_indices(B, M, self.n_negatives).numpy(), dev).view(B, M, self.n_negatives)

        x = Fn.W2VGather.apply(x, idx, inv)
        x = Fn.Linear.apply(x, self.final_proj.weight, self.final_proj.bias, p)
        logits = Fn.W2VLogits.apply(x, y, neg, float(self.logit_temp))

        out = {"x": logits, "padding_mask": padding_mask, "features_pen": features_pen}
        out.update(result)
        if prob_ppl is not None:
            out["prob_perplexity"] = prob_ppl
            out["code_perplexity"] = code_ppl
            out["num_vars"] = num_vars
            out["temp"] = curr_temp
        return out

    def get_logits(self, net_output):
        logits = net_output["x"]
        logits = logits.transpose(0, 2)
        return logits.reshape(-1, logits.size(-1))

    def get_targets(self, sample, net_output, expand_steps=True):
        x = net_output["x"]
        return x.new_zeros(x.size(1) * x.size(2), dtype=torch.long)

    def get_extra_losses(self, net_output):
        pen = []
        if "prob_perplexity" in net_output:
            pen.append((net_output["num_vars"] - net_output["prob_perplexity"]) / net_output["num_vars"])
        if "features_pen" in net_output:
            pen.append(net_output["features_pen"])
        return pen


class ConstrastiveCriterion(nn.Module):
    """rnnt/wav2vec.py:424-528: returns (loss, sample_size, logging_output) with the reference's keys and values.  The
    cross-entropy runs Fn.W2VCrossEntropy on the device; the whole logging_output comes from one device-to-host copy.
    Only infonce=True (what cli/pretrain_wav2vec.py passes) is implemented."""

    def __init__(self, infonce=False, loss_weights=None, log_keys=None):
        super().__init__()
        self.infonce = infonce
        self.loss_weights = loss_weights
        self.log_keys = [] if log_keys is None else log_keys

    def forward(self, model, sample, reduce=True):
        if not self.infonce:
            raise ValueError("ConstrastiveCriterion: infonce=False is not supported")
        if self.loss_weights is not None:
            n_extra = int(model.quantizer is not None or model.input_quantizer is not None) + 1
            if len(self.loss_weights) == 1 and n_extra != 1:
                self.loss_weights = [self.loss_weights[0]] * n_extra
            if len(self.loss_weights) != n_extra:
                raise ValueError("ConstrastiveCriterion: %d loss weights for %d extra losses (the reference's assertion)"
                                 % (len(self.loss_weights), n_extra))
        results = model(sample)
        logits = results["x"]
        loss, correct = Fn.W2VCrossEntropy.apply(logits)
        sample_size = logits.shape[1] * logits.shape[2]
        losses = [loss.detach()]
        if self.loss_weights is not None:
            for p, coef in zip(model.get_extra_losses(results), self.loss_weights):
                if coef != 0 and p is not None:
                    p = coef * p.float() * sample_size
                    loss = loss + p
                    losses.append(p.detach())

        host_keys, vals = [], []
        for lk in self.log_keys:
            if lk in ("logits", "target") or lk not in results:
                continue
            if isinstance(results[lk], torch.Tensor):
                host_keys.append(lk)
                vals.append(results[lk].detach().float().reshape(()))
        dev = torch.stack([loss.detach()] + losses + [correct] + vals).cpu().tolist()       # the one readback

        logging_output = {"loss": dev[0], "ntokens": sample_size, "sample_size": sample_size}
        for lk in self.log_keys:
            if lk == "logits":
                if not self.training:
                    logging_output["logits"] = model.get_logits(results).float().cpu().numpy()
            elif lk == "target":
                if not self.training:
                    logging_output["target"] = model.get_targets(None, results).cpu().numpy()
            elif lk in results:
                logging_output[lk] = (dev[2 + len(losses) + host_keys.index(lk)] if lk in host_keys
                                      else float(results[lk]))
        if len(losses) > 1:
            for i in range(len(losses)):
                logging_output[f"loss_{i}"] = dev[1 + i]
        logging_output["correct"] = int(dev[1 + len(losses)])
        logging_output["count"] = sample_size
        return loss, sample_size, logging_output
