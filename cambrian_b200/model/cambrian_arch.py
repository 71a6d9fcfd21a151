"""Multimodal glue — H100-native mirror of the reference's `cambrian/model/cambrian_arch.py`.

`CambrianMetaModel` builds the same sub-modules with the same attribute / state-dict names (mm_projector,
mm_projector_aux_{i}, vision_sampler_{g}, vision_sampler_layers, vision_query, image_newline; cambrian_arch.py:35-87,
:99-200) and `CambrianMetaForCausalLM.prepare_inputs_labels_for_multimodal` reproduces the static-shape branch the
reference trains with (cambrian_arch.py:340-490, the `IS_XLA_AVAILABLE` side): towers -> aux projectors -> global
context -> connector SVA -> mm_projector -> newline column -> splice into the token embeddings.

Differences that are purely layout, not semantics:
  * the per-query window gather (`rearrange_vision_tower_features_train`, :271-287) is NOT materialised: the aux
    feature grids stay in their natural [B, N_i, 1024] layout and the SVA kernels do the index arithmetic;
  * embedding lookup + image-span replacement + newline append are one gather kernel (`EmbedSpliceFn`).
The per-sample dynamic-shape branch the reference runs off-XLA (:289-330, :422-451, :493-609; SURVEY.md §8f rank 3) is
`_prepare_dynamic`: taken when `image_sizes` holds a non-square image (square images give identical results on both
branches), inference only.  There the windows ARE materialised (`cb_window_gather`, with the `unpad_image` crop) because
the per-sample query counts differ, and the ragged splice is one gather kernel driven by a host-built row map.
"""
from __future__ import annotations

from abc import ABC, abstractmethod

import torch
import torch.nn as nn

from .. import ops
from ..autograd import EmbedSpliceFn, ExpandRowsFn, MeanTokensFn, ResizeTokenGridFn, _await
from .multimodal_encoder.builder import build_vision_tower_aux_list
from .multimodal_projector.builder import CBGELU, CBLayerNorm, CBLinear, build_vision_projector
from .vision_sampler import VisionTokenSampler

IGNORE_INDEX = -100
IMAGE_TOKEN_INDEX = -200
_TOWER_STREAMS = __import__("os").environ.get("CB_TOWER_STREAMS", "1") != "0"


def _kv_sizes(aux_token_lens, query_num):
    return [int(t ** 0.5) // int(query_num ** 0.5) for t in aux_token_lens]


class CambrianMetaModel:
    def __init__(self, config):
        super(CambrianMetaModel, self).__init__(config)
        if hasattr(config, "mm_vision_tower_aux_list"):
            self._build_vision_modules(config, delay_load=True)

    def _build_vision_modules(self, config, delay_load):
        projector_type = getattr(config, "mm_projector_type", "linear")
        self.vision_tower_aux_list = build_vision_tower_aux_list(config, delay_load=delay_load)
        if projector_type == "sva":
            vh = config.vision_hidden_size
            G = config.num_query_group
            self.mm_projector = nn.Sequential(CBLinear(vh * G, config.hidden_size), CBGELU(),
                                              CBLinear(config.hidden_size, config.hidden_size))
            aux_lens = config.mm_vision_tower_aux_token_len_list
            for i, tower in enumerate(self.vision_tower_aux_list):
                setattr(self, f"mm_projector_aux_{i}",
                        nn.Sequential(CBLinear(tower.hidden_size, vh), CBGELU(), CBLinear(vh, vh), CBLayerNorm(vh)))
            T = len(self.vision_tower_aux_list)
            for g in range(G):
                setattr(self, f"vision_sampler_{g}",
                        VisionTokenSampler(vh, vh, [vh] * T, _kv_sizes(aux_lens, config.query_num_list[g]), vh,
                                           config.connector_depth))
            if not config.connector_only:
                sizes = _kv_sizes(aux_lens, config.image_token_len)
                self.vision_sampler_layers = nn.ModuleList([
                    VisionTokenSampler(config.hidden_size, vh, [vh] * T, sizes, vh, 1)
                    for _ in range(config.num_of_vision_sampler_layers)])
            self.vision_query = nn.Parameter(torch.randn((G, vh)) * (1.0 / vh) ** 0.5)      # :161-164
            self.image_newline = nn.Parameter(torch.randn(config.hidden_size) * (1.0 / config.hidden_size) ** 0.5)
        else:
            config.mm_hidden_size = sum(t.hidden_size for t in self.vision_tower_aux_list)
            self.mm_projector = build_vision_projector(config)
            self.image_newline = nn.Parameter(torch.randn(config.hidden_size) * (1.0 / config.hidden_size) ** 0.5)

    def get_vision_tower_aux_list(self):
        return getattr(self, "vision_tower_aux_list", None)

    def initialize_vision_modules(self, model_args, fsdp=None):
        """cambrian_arch.py:99-200: copy the SVA hyper-parameters onto config, build towers and connector modules."""
        cfg = self.config
        cfg.mm_vision_tower_aux_list = model_args.vision_tower_aux_list
        cfg.mm_vision_tower_aux_token_len_list = model_args.vision_tower_aux_token_len_list
        cfg.image_token_len = getattr(model_args, "image_token_len", 576)
        cfg.mm_projector_type = getattr(model_args, "mm_projector_type", "sva")
        cfg.mm_vision_select_layer = getattr(model_args, "mm_vision_select_layer", -2)
        cfg.mm_vision_select_feature = getattr(model_args, "mm_vision_select_feature", "patch")
        cfg.use_mm_proj = True
        if cfg.mm_projector_type == "sva":
            cfg.vision_hidden_size = model_args.vision_hidden_size
            cfg.num_query_group = model_args.num_query_group
            cfg.query_num_list = model_args.query_num_list
            assert cfg.num_query_group == len(cfg.query_num_list)                              # :117
            cfg.connector_depth = model_args.connector_depth
            cfg.connector_only = model_args.connector_only
            cfg.num_of_vision_sampler_layers = getattr(model_args, "num_of_vision_sampler_layers", 0)
            cfg.start_of_vision_sampler_layers = getattr(model_args, "start_of_vision_sampler_layers", 0)
            cfg.stride_of_vision_sampler_layers = getattr(model_args, "stride_of_vision_sampler_layers", 1)
        self._build_vision_modules(cfg, delay_load=False)
        adapter = getattr(model_args, "pretrain_mm_mlp_adapter", None)
        if adapter is not None:                                                                 # :183-200
            from ..checkpoint import load_mm_projector
            weights = torch.load(adapter, map_location="cpu")
            prefix = "" if any(k.startswith("model.") for k in weights) else "model."

            class _Wrap:                                   # the adapter file is keyed from the ForCausalLM root
                def __init__(self, inner):
                    self.inner = inner

                def state_dict(self):
                    return {"model." + k: v for k, v in self.inner.state_dict().items()}
            load_mm_projector(_Wrap(self), {prefix + k: v for k, v in weights.items()}, strict_submodules=True)


class WindowedFeatures(list):
    """Marks a list of tower features as ALREADY window-rearranged ([sum_b h_b*w_b, r_i^2, C], the layout the
    reference's non-XLA branch hands to the decoder loop) as opposed to the natural [B, N_i, C] grids the static
    branch keeps."""


def unmask_attention_mask(mask, original_size):
    """cambrian_arch.py:203-227 — zero the letter-box band of a [1, h, w] mask (in place), host tensor."""
    original_w, original_h = original_size
    cur_h, cur_w = mask.shape[1:3]
    if original_w / original_h > cur_w / cur_h:
        new_height = int(original_h * (cur_w / original_w))
        padding = (cur_h - new_height) // 2
        if padding > 0:
            mask[:, :padding, :] = 0
            mask[:, -padding:, :] = 0
    else:
        new_width = int(original_w * (cur_h / original_h))
        padding = (cur_w - new_width) // 2
        if padding > 0:
            mask[:, :, :padding] = 0
            mask[:, :, -padding:] = 0
    return mask


def unpad_bounds(cur_h, cur_w, original_size):
    """The crop `unpad_image` (cambrian_arch.py:230-256) applies to dims (1, 2) of its argument: (y0, y1, x0, x1)."""
    original_w, original_h = original_size
    if original_w / original_h > cur_w / cur_h:
        new_height = int(original_h * (cur_w / original_w))
        padding = (cur_h - new_height) // 2
        return padding, cur_h - padding, 0, cur_w
    new_width = int(original_w * (cur_h / original_h))
    padding = (cur_w - new_width) // 2
    return 0, cur_h, padding, cur_w - padding


def unpad_image(tensor, original_size):
    """cambrian_arch.py:230-256 (any tensor whose dims 1, 2 are the padded grid)."""
    y0, y1, x0, x1 = unpad_bounds(tensor.shape[1], tensor.shape[2], original_size)
    return tensor[:, y0:y1, x0:x1]


def _window_masks_inference(aux_side, q_side, image_size, unpad):
    """Host part of rearrange_vision_tower_features_inference (cambrian_arch.py:306-320) for one sample."""
    r = aux_side // q_side
    m = torch.ones((1, aux_side, aux_side), dtype=torch.bool)
    m = unmask_attention_mask(m, image_size)
    m = m.view(1, q_side, r, q_side, r).permute(0, 1, 3, 2, 4).contiguous()
    if unpad:
        m = unpad_image(m, image_size)
    m = m.flatten(0, 2).flatten(1, 2).clone()
    m[m.sum(-1) == 0] = True
    return m


class CambrianMetaForCausalLM(ABC):
    @abstractmethod
    def get_model(self):
        pass

    def get_vision_tower_aux_list(self):
        return self.get_model().get_vision_tower_aux_list()

    def encode_images(self, image_aux_list):
        """cambrian_arch.py:332-338.  The towers are independent of each other (and frozen in every released recipe), so
        each runs on its own CUDA stream: most ViT GEMMs are a wave and a bit on 132 SMs (M = B * 577 rows -> ~150 tiles),
        and with one-CTA-per-tile grids the idle SMs of one tower's last wave take tiles of another tower's kernel instead
        of waiting (CB_TOWER_STREAMS=0 runs them back to back on the current stream)."""
        towers = self.get_model().get_vision_tower_aux_list()
        imgs = list(image_aux_list)
        multi = (_TOWER_STREAMS and len(towers) > 1 and all(torch.is_tensor(i) and i.is_cuda for i in imgs)
                 and not any(getattr(t, "unfreeze_mm_vision_tower", False) for t in towers))
        if not multi:
            return [tower(img) for img, tower in zip(imgs, towers)]
        main = torch.cuda.current_stream()
        pool = getattr(self, "_tower_streams", None)
        if pool is None or len(pool) < len(towers) or pool[0].device != imgs[0].device:
            pool = [torch.cuda.Stream(device=imgs[0].device) for _ in towers]
            self._tower_streams = pool
        # the largest tower first: its big GEMMs are the backdrop the small ones fill into
        order = sorted(range(len(towers)), key=lambda i: -imgs[i].shape[-1])
        outs = [None] * len(towers)
        for i in order:
            st = pool[i]
            st.wait_stream(main)                      # inputs (H2D copies, casts) were produced on the current stream
            with torch.cuda.stream(st):
                outs[i] = towers[i](imgs[i])
        for i in order:
            main.wait_stream(pool[i])
            if torch.is_tensor(outs[i]):
                outs[i].record_stream(main)           # allocated on the side stream, consumed (and freed) on the main one
            if torch.is_tensor(imgs[i]):
                imgs[i].record_stream(pool[i])
        return outs

    def rearrange_vision_tower_features_train(self, vision_tower_aux_feature_list, vision_tower_aux_attention_masks_list,
                                              query_side_len):
        """cambrian_arch.py:271-287: [B, (q r)^2, C] -> [B q^2, r^2, C]; masks -> [B q^2, r^2]."""
        feats, masks = [], []
        for f, m in zip(vision_tower_aux_feature_list, vision_tower_aux_attention_masks_list):
            w = ops.window_gather(f.to(torch.bfloat16).contiguous(), query_side_len)
            feats.append(w)
            masks.append(m.view(w.shape[0], w.shape[1]))
        return feats, masks

    def rearrange_vision_tower_features_inference(self, vision_tower_aux_feature_list, query_side_len, image_sizes,
                                                  unpad=False):
        """cambrian_arch.py:289-330: per-sample windows (+ the `unpad_image` crop of the q x q window grid) and the
        letter-box masks derived from the ORIGINAL image sizes; samples are concatenated along dim 0 (ragged)."""
        feats, masks = WindowedFeatures(), []
        bs = vision_tower_aux_feature_list[0].shape[0]
        for f in vision_tower_aux_feature_list:
            f = f.to(torch.bfloat16).contiguous()
            aux_side = int(f.shape[1] ** 0.5)
            assert (aux_side // query_side_len) * query_side_len == aux_side                       # :296
            fw, mw = [], []
            for b in range(bs):
                crop = unpad_bounds(query_side_len, query_side_len, image_sizes[b]) if unpad else None
                fw.append(ops.window_gather(f[b:b + 1], query_side_len, crop))
                mw.append(_window_masks_inference(aux_side, query_side_len, image_sizes[b], unpad))
            feats.append(fw[0] if bs == 1 else torch.cat(fw, 0))
            masks.append(torch.cat(mw, 0).to(f.device, non_blocking=True))
        return feats, masks

    def _prepare_dynamic(self, input_ids, position_ids, attention_mask, past_key_values, labels, images, image_sizes):
        """The reference's non-XLA branch (cambrian_arch.py:387-389, :422-451, :493-609): per-sample unpadded query
        grids for non-square images.  Inference only (no backward through the gather kernels)."""
        model = self.get_model()
        cfg = model.config
        if torch.is_grad_enabled() and any(p.requires_grad for p in model.parameters()):
            raise NotImplementedError("the dynamic-shape (non-square image) branch is inference-only: run under torch.no_grad()")
        sync = getattr(self, "_cb_param_sync", None)
        if sync is not None:
            sync()
        bs = images[0].shape[0]
        q_num = cfg.image_token_len
        fh = fw = int(q_num ** 0.5)
        feats = self.encode_images(images)
        feats_final = masks_final = ctx_final = None
        if cfg.mm_projector_type == "sva":
            aux = [getattr(model, f"mm_projector_aux_{i}")(f.to(torch.bfloat16)) for i, f in enumerate(feats)]
            ctx = MeanTokensFn.apply(aux[0])                                                     # [B, vh]
            outs = []
            for g, query_num in enumerate(cfg.query_num_list):
                qs = int(query_num ** 0.5)
                n = bs * query_num
                _await(model.vision_query)
                queries = ExpandRowsFn.apply(model.vision_query[g:g + 1].to(torch.bfloat16), n)
                ctx_g = ExpandRowsFn.apply(ctx, query_num)
                f_i, m_i = self.rearrange_vision_tower_features_inference(aux, qs, image_sizes)     # :389
                qf = getattr(model, f"vision_sampler_{g}")(queries.view(n, 1, -1), ctx_g.view(n, 1, -1), *f_i, *m_i)
                qf = qf.view(bs, query_num, -1)
                if qs != fh:                                                                       # :394-401
                    qf = ResizeTokenGridFn.apply(qf, qs, fh)
                outs.append(qf)
            image_features = outs[0] if len(outs) == 1 else torch.cat(outs, -1)
            feats_final, masks_final = self.rearrange_vision_tower_features_inference(aux, fh, image_sizes, unpad=True)
        else:
            image_features = (feats[0] if len(feats) == 1 else torch.cat(feats, -1)).to(torch.bfloat16)
        image_features = model.mm_projector(image_features).contiguous()                          # [bs, fh*fw, H]
        bounds = [unpad_bounds(fh, fw, image_sizes[b]) for b in range(bs)]
        final_size = [(y1 - y0, x1 - x0) for (y0, y1, x0, x1) in bounds]
        if cfg.mm_projector_type == "sva":
            ctx_final = torch.cat([ExpandRowsFn.apply(ctx[b:b + 1], h * w) for b, (h, w) in enumerate(final_size)], 0)
            ctx_final = ctx_final.view(-1, 1, ctx.shape[-1])
        # ---- ragged splice, host side (cambrian_arch.py:493-609) -> one row map for the gather kernel
        NEWLINE = -(2 ** 31)
        dev = input_ids.device
        ids_cpu = input_ids.detach().to("cpu")
        _labels, _position_ids, _attention_mask = labels, position_ids, attention_mask
        am = torch.ones_like(ids_cpu, dtype=torch.bool) if attention_mask is None else attention_mask.detach().to("cpu").bool()
        lab_cpu = torch.full_like(ids_cpu, IGNORE_INDEX) if labels is None else labels.detach().to("cpu")
        rows_src, rows_lab = [], []
        cur_image_idx = 0

        def image_rows(k):
            y0, y1, x0, x1 = bounds[k]
            r = []
            for y in range(y0, y1):
                r.extend(-2 - (k * fh * fw + y * fw + x) for x in range(x0, x1))
                r.append(NEWLINE)
            return r

        for b in range(bs):
            cur = ids_cpu[b][am[b]].tolist()
            cl = lab_cpu[b][am[b]].tolist()
            src, lab = [], []
            if IMAGE_TOKEN_INDEX not in cur:
                cur_image_idx += 1                                                                  # :519-526
                rows_src.append(cur)
                rows_lab.append(cl)
                continue
            for t, l in zip(cur, cl):
                if t == IMAGE_TOKEN_INDEX:
                    ir = image_rows(cur_image_idx)
                    cur_image_idx += 1
                    src.extend(ir)
                    lab.extend([IGNORE_INDEX] * len(ir))
                else:
                    src.append(t)
                    lab.append(l)
            rows_src.append(src)
            rows_lab.append(lab)
        max_tok = getattr(cfg, "tokenizer_model_max_length", None)
        if max_tok is not None:
            rows_src = [r[:max_tok] for r in rows_src]
            rows_lab = [r[:max_tok] for r in rows_lab]
        max_len = max(len(r) for r in rows_src)
        left = getattr(cfg, "tokenizer_padding_side", "right") == "left"
        src_map = torch.full((bs, max_len), -1, dtype=torch.int32)
        new_labels = torch.full((bs, max_len), IGNORE_INDEX, dtype=lab_cpu.dtype)
        new_mask = torch.zeros((bs, max_len), dtype=torch.bool)
        new_pos = torch.zeros((bs, max_len), dtype=torch.long)
        for b, (r, l) in enumerate(zip(rows_src, rows_lab)):
            n = len(r)
            if n == 0:
                continue
            sl = slice(max_len - n, max_len) if left else slice(0, n)
            src_map[b, sl] = torch.tensor(r, dtype=torch.int32)
            new_labels[b, sl] = torch.tensor(l, dtype=lab_cpu.dtype)
            new_mask[b, sl] = True
            new_pos[b, sl] = torch.arange(n)
        new_embeds = ops.embed_splice_ragged(model.embed_tokens.weight, image_features.view(-1, image_features.shape[-1]),
                                             model.image_newline, src_map.view(-1).to(dev), bs, max_len)
        new_labels = None if _labels is None else new_labels.to(dev)
        out_mask = None if _attention_mask is None else new_mask.to(dev).to(_attention_mask.dtype)
        out_pos = None if _position_ids is None else new_pos.to(dev)
        return (None, out_pos, out_mask, past_key_values, new_embeds, new_labels, feats_final, masks_final, final_size,
                ctx_final)

    def prepare_inputs_labels_for_multimodal(self, input_ids, position_ids, attention_mask, past_key_values, labels,
                                             images, image_aux_attention_masks_list=None, image_sizes=None,
                                             image_positions=None):
        """`image_positions` (extension, host ints): index of the <image> indicator of every sample of an ALREADY
        expanded batch (what the collator knows); skips the device->host scan of input_ids (a stream sync)."""
        model = self.get_model()
        towers = model.get_vision_tower_aux_list()
        if towers is None or images is None or input_ids.shape[1] == 1:                          # :345-346
            return input_ids, position_ids, attention_mask, past_key_values, None, labels, None, None, None, None
        cfg = model.config
        bs = images[0].shape[0]
        q_num = cfg.image_token_len
        q_side = int(q_num ** 0.5)
        if image_sizes is not None and any(int(w) != int(h) for (w, h) in image_sizes):
            # per-sample unpadded grids: the reference's non-XLA branch (for square images it reduces to the static one)
            return self._prepare_dynamic(input_ids, position_ids, attention_mask, past_key_values, labels, images,
                                         image_sizes)
        span = q_num + q_side
        # --- locate the image span of every sample; expand a bare <image> indicator the way the collator does
        #     (train_fsdp.py:1089-1165) when the caller passes un-expanded ids (inference path)
        img_start = None
        if image_positions is not None:
            starts = [int(p) for p in image_positions]
        elif getattr(cfg, "inputs_pre_expanded", False):
            # the static-shape contract of the reference's training branch (IS_XLA_AVAILABLE side, cambrian_arch.py:457-490):
            # the collator has already expanded <image> into the 600-slot span (train_fsdp.py:1089-1165).  The span start is
            # then located ON THE DEVICE (index plumbing, no host sync); samples without an image get -1.
            hit = input_ids == IMAGE_TOKEN_INDEX
            img_start = torch.where(hit.any(1), hit.int().argmax(1), torch.full((bs,), -1, device=input_ids.device,
                                                                                dtype=torch.long)).to(torch.int32)
        else:
            ids_cpu = input_ids.detach().to("cpu")
            if any(int((row == IMAGE_TOKEN_INDEX).sum()) > 1 for row in ids_cpu):
                raise NotImplementedError("exactly one image per sample (train_fsdp.py:1100)")
            flags = []          # per row with an image: is the <image> indicator still bare (needs the 600-slot expansion)?
            for row in ids_cpu:
                pos = torch.where(row == IMAGE_TOKEN_INDEX)[0]
                if len(pos) == 1:
                    p0 = int(pos[0])
                    flags.append(p0 + span > row.shape[0] or bool((row[p0 + 1:p0 + span] != 0).any()))
            if any(flags) and not all(flags):
                raise ValueError("a batch must hold either collator-expanded image spans or bare <image> indicators, not a "
                                 "mix (pass image_positions, or expand every row)")
            needs_expand = any(flags)
            if needs_expand:
                input_ids, labels, attention_mask, position_ids = _expand_image_tokens(
                    ids_cpu, labels, attention_mask, span, input_ids.device)
                ids_cpu = input_ids.detach().to("cpu")
            starts = []
            for row in ids_cpu:
                pos = torch.where(row == IMAGE_TOKEN_INDEX)[0]
                starts.append(int(pos[0]) if len(pos) else -1)
        if img_start is None:
            img_start = torch.tensor(starts, dtype=torch.int32).to(input_ids.device, non_blocking=True)

        feats = self.encode_images(images)                                                      # :366
        # (TrainEngine: the optimizer of the previous step may still be running on its side stream under the frozen towers
        #  above; every trainable block below waits for exactly its own bucket — autograd._await)
        feats_final = masks_final = ctx_final = None
        if cfg.mm_projector_type == "sva":
            aux = [getattr(model, f"mm_projector_aux_{i}")(f.to(torch.bfloat16)) for i, f in enumerate(feats)]   # :372-379
            ctx = MeanTokensFn.apply(aux[0])                                                    # :377  [B, vh]
            T = len(aux)
            outs = []
            for g, query_num in enumerate(cfg.query_num_list):
                qs = int(query_num ** 0.5)
                n = bs * query_num
                _await(model.vision_query)
                queries = ExpandRowsFn.apply(model.vision_query[g:g + 1].to(torch.bfloat16), n)      # :383
                ctx_g = ExpandRowsFn.apply(ctx, query_num)                                           # :384
                masks = _masks_for(image_aux_attention_masks_list, aux, qs, n)
                sampler = getattr(model, f"vision_sampler_{g}")
                qf = sampler(queries.view(n, 1, -1), ctx_g.view(n, 1, -1), *aux, *masks, natural_layout=(bs, qs))
                qf = qf.view(bs, query_num, -1)
                if qs != q_side:                                                                     # :394-401
                    qf = ResizeTokenGridFn.apply(qf, qs, q_side)
                outs.append(qf)
            image_features = outs[0] if len(outs) == 1 else torch.cat(outs, -1)
            feats_final = aux                                                                    # natural layout
            masks_final = _masks_for(image_aux_attention_masks_list, aux, q_side, bs * q_num)
            ctx_final = ExpandRowsFn.apply(ctx, q_num).view(bs * q_num, 1, -1)                   # :406
        else:
            image_features = feats[0] if len(feats) == 1 else torch.cat(feats, -1)              # :408
            image_features = image_features.to(torch.bfloat16)
        image_features = model.mm_projector(image_features)                                     # :410-411
        meta = dict(ids=input_ids.contiguous(), img_start=img_start, q_side=q_side,
                    params=(model.embed_tokens.weight, model.image_newline))
        inputs_embeds = EmbedSpliceFn.apply(meta, model.embed_tokens.weight, image_features.contiguous(),
                                            model.image_newline)
        final_size = [(q_side, q_side)] * bs
        return (None, position_ids, attention_mask, past_key_values, inputs_embeds, labels, feats_final, masks_final,
                final_size, ctx_final)


def _masks_for(mask_list, aux, q_side, n):
    """image_aux_attention_masks_list entries are [B*q^2, r_i^2] bool (collator, train_fsdp.py:1122-1137) or absent."""
    if mask_list is None:
        return [None] * len(aux)
    out = []
    for m, a in zip(mask_list, aux):
        r = int(a.shape[1] ** 0.5) // q_side
        out.append(None if m is None else m.reshape(n, r * r))
    return out


def _expand_image_tokens(ids_cpu, labels, attention_mask, span, device):
    """Host-side mirror of the collator's placeholder expansion (train_fsdp.py:1102-1150) for un-expanded inputs:
    the single -200 id becomes -200 followed by span-1 zero ids; labels get IGNORE_INDEX; positions run on."""
    new_ids, new_labels, new_mask = [], [], []
    lab_cpu = labels.detach().to("cpu") if labels is not None else None
    msk_cpu = attention_mask.detach().to("cpu") if attention_mask is not None else None
    for b, row in enumerate(ids_cpu):
        pos = torch.where(row == IMAGE_TOKEN_INDEX)[0]
        if len(pos) == 0:
            pad = span - 1
            new_ids.append(torch.cat([row, torch.zeros(pad, dtype=row.dtype)]))
            new_labels.append(None if lab_cpu is None else torch.cat([lab_cpu[b], torch.full((pad,), IGNORE_INDEX)]))
            m = torch.ones_like(row, dtype=torch.bool) if msk_cpu is None else msk_cpu[b].bool()
            new_mask.append(torch.cat([m, torch.zeros(pad, dtype=torch.bool)]))
            continue
        p0 = int(pos[0])
        new_ids.append(torch.cat([row[:p0 + 1], torch.zeros(span - 1, dtype=row.dtype), row[p0 + 1:]]))
        if lab_cpu is not None:
            new_labels.append(torch.cat([lab_cpu[b][:p0], torch.full((span,), IGNORE_INDEX), lab_cpu[b][p0 + 1:]]))
        m = torch.ones_like(row, dtype=torch.bool) if msk_cpu is None else msk_cpu[b].bool()
        new_mask.append(torch.cat([m[:p0], torch.ones(span, dtype=torch.bool), m[p0 + 1:]]))
    ids = torch.stack(new_ids).to(device)
    lab = torch.stack(new_labels).to(device) if lab_cpu is not None else None
    mask = torch.stack(new_mask).to(device)
    pos_ids = (mask.long().cumsum(1) - 1).clamp_(min=0)
    return ids, lab, mask, pos_ids
