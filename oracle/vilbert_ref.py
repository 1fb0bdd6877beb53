"""CPU ORACLE -- TEST INFRASTRUCTURE ONLY.  PARITY UNPINNED.

Plain-PyTorch fp32 restatement of the hot path the reference worker calls once per
request: ``model(question, features, spatials, segment_ids, input_mask, image_mask,
co_attention_mask, task_tokens, output_all_attention_masks=True)``
(worker.py:286-289) on the object built at worker.py:530-536
(``VILBertForVLTasks.from_pretrained(..., config=config, num_labels=3129)``).

The arithmetic itself lives in the third-party package ``vilbert`` (upstream
facebookresearch/vilbert-multi-task, ``vilbert/vilbert.py``), imported at worker.py:44-46.
It is un-vendored, un-pinned (absent from requirements.txt:1-69, ``.SUBMODULES.json:8`` has no
submodules) and not installed here, and the reference holds no test, golden vector or checkpoint
for this path (demo/tests.py:1-3 is an empty stub).  This file therefore restates the *published*
algorithm (arXiv:1908.02265 section 3, arXiv:1912.02315) constrained by every in-tree call site;
there is nothing in the reference tree to pin it against numerically  ==>  "parity unpinned".
The one number the tree does pin -- "270 million" parameters (README.md:4) -- is checked by
``count_parameters`` (268.0 M unique parameters, the tied LM decoder counted once).  Three pieces are additionally
cross-checked against independent implementations (tests/test_oracle.py): the text ``BertLayer`` and ``BertEmbeddings`` against
HuggingFace ``transformers``, both directions of the co-attention against ``torch.nn.MultiheadAttention``.

Only ``tests/``, ``__graft_entry__.smoke()`` and the ``cpu_baseline`` / ``--impl reference`` legs of
``bench.py`` may import this module; the product path (``vilbert_b200``) never does.

Every [UPSTREAM] assumption that no in-tree line can confirm is a named flag in ``UPSTREAM_ASSUMPTIONS``.
State-dict key names are the upstream ones (SURVEY.md section 8b) so a real
``pytorch_model_9.bin`` (worker.py:470) loads into this module with ``load_state_dict``.
"""
from __future__ import annotations

import copy
import json
import math
from typing import Dict, List, Optional

import torch
from torch import nn

# --------------------------------------------------------------------------------------------
# Named [UPSTREAM] assumptions (each is a behaviour of vilbert/vilbert.py that the in-tree code
# only constrains indirectly).  Tests print this table next to every parity number.
# --------------------------------------------------------------------------------------------
UPSTREAM_ASSUMPTIONS = {
    "task_token_position": 1,            # task embedding row inserted after [CLS]; worker.py:516-517 enables it
    "task_token_gets_pos_type_emb": False,  # inserted row is the bare task embedding (cat happens after the sum)
    "text_mask_prepends_one": True,      # attention_mask <- cat([1], attention_mask) when task tokens are on
    "additive_mask_value": -10000.0,     # (1 - mask) * -10000 on attention scores and on vision_logit
    "co_attention_mask_used": False,     # built (x5) but its use is commented out upstream; worker passes zeros (worker.py:455)
    "bi_ctx_for_text": "softmax(Q_text K_img^T / sqrt(d) + img_mask) V_img",
    "bi_ctx_for_image": "softmax(Q_img K_text^T / sqrt(d) + txt_mask) V_text",
    "bioutput_q_dense_unused": True,     # q_dense1/q_dense2 exist in the checkpoint, never applied
    "layer_schedule": "T0-5 C0 (T6 V0 C1) ... (T10 V4 C5) V5 T11",
    "gelu": "erf",                       # x * 0.5 * (1 + erf(x / sqrt(2)))
    "layernorm_eps": 1e-12,
    "fusion": "mul",                     # pooled = pooled_t * pooled_v
    "pooler_activation": "relu",
    "binary_head_when_batch_odd": "bi_seq_relationship score",  # element 3 of the tuple if B is odd
}

DEFAULT_CONFIG: Dict = {
    # [UPSTREAM] config/bert_base_6layer_6conect.json (file name pinned by worker.py:472)
    "attention_probs_dropout_prob": 0.1,
    "hidden_act": "gelu",
    "hidden_dropout_prob": 0.1,
    "hidden_size": 768,
    "initializer_range": 0.02,
    "intermediate_size": 3072,
    "max_position_embeddings": 512,
    "num_attention_heads": 12,
    "num_hidden_layers": 12,
    "type_vocab_size": 2,
    "vocab_size": 30522,
    "v_feature_size": 2048,
    "v_target_size": 1601,
    "v_hidden_size": 1024,
    "v_num_hidden_layers": 6,
    "v_num_attention_heads": 8,
    "v_intermediate_size": 1024,
    "bi_hidden_size": 1024,
    "bi_num_attention_heads": 8,
    "bi_intermediate_size": 1024,
    "bi_attention_type": 1,
    "v_attention_probs_dropout_prob": 0.1,
    "v_hidden_act": "gelu",
    "v_hidden_dropout_prob": 0.1,
    "v_initializer_range": 0.02,
    "v_biattention_id": [0, 1, 2, 3, 4, 5],
    "t_biattention_id": [6, 7, 8, 9, 10, 11],
    "pooling_method": "mul",
    "fusion_method": "mul",
    # mutated by the worker after loading (worker.py:509-522)
    "predict_feature": False,
    "task_specific_tokens": True,
    "dynamic_attention": False,
    "visualization": True,
    "num_task_tokens": 20,
}


class RefConfig:
    """Attribute bag with the fields of the upstream BertConfig (worker.py:495, 506-522)."""

    def __init__(self, **kw):
        d = copy.deepcopy(DEFAULT_CONFIG)
        d.update(kw)
        self.__dict__.update(d)

    @classmethod
    def from_json_file(cls, path):
        with open(path, "r", encoding="utf-8") as f:
            return cls(**json.load(f))

    def to_dict(self):
        return copy.deepcopy(self.__dict__)


def gelu(x):
    return x * 0.5 * (1.0 + torch.erf(x / math.sqrt(2.0)))


class BertLayerNorm(nn.Module):
    """TF-style LayerNorm, epsilon inside the square root; eps=1e-12 everywhere upstream."""

    def __init__(self, hidden_size, eps=1e-12):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(hidden_size))
        self.bias = nn.Parameter(torch.zeros(hidden_size))
        self.variance_epsilon = eps

    def forward(self, x):
        u = x.mean(-1, keepdim=True)
        s = (x - u).pow(2).mean(-1, keepdim=True)
        x = (x - u) / torch.sqrt(s + self.variance_epsilon)
        return self.weight * x + self.bias


class GeLU(nn.Module):
    def forward(self, x):
        return gelu(x)


# ------------------------------------------------------------------ embeddings (SURVEY a-2, a-3)
class BertEmbeddings(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.task_specific_tokens = c.task_specific_tokens
        self.word_embeddings = nn.Embedding(c.vocab_size, c.hidden_size, padding_idx=0)
        self.position_embeddings = nn.Embedding(c.max_position_embeddings, c.hidden_size)
        self.token_type_embeddings = nn.Embedding(c.type_vocab_size, c.hidden_size)
        self.LayerNorm = BertLayerNorm(c.hidden_size, eps=1e-12)
        if self.task_specific_tokens:
            self.task_embeddings = nn.Embedding(c.num_task_tokens, c.hidden_size)

    def forward(self, input_ids, token_type_ids, task_ids):
        seq_length = input_ids.size(1)
        position_ids = torch.arange(seq_length, dtype=torch.long, device=input_ids.device)
        position_ids = position_ids.unsqueeze(0).expand_as(input_ids)
        e = (self.word_embeddings(input_ids) + self.position_embeddings(position_ids)
             + self.token_type_embeddings(token_type_ids))
        if self.task_specific_tokens:
            task = self.task_embeddings(task_ids)                      # [B,1,H]
            e = torch.cat([e[:, 0:1], task, e[:, 1:]], dim=1)          # task row at index 1
        return self.LayerNorm(e)                                        # dropout = identity (model.eval(), worker.py:534)


class BertImageEmbeddings(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.image_embeddings = nn.Linear(c.v_feature_size, c.v_hidden_size)
        self.image_location_embeddings = nn.Linear(5, c.v_hidden_size)
        self.LayerNorm = BertLayerNorm(c.v_hidden_size, eps=1e-12)

    def forward(self, feats, loc):
        return self.LayerNorm(self.image_embeddings(feats) + self.image_location_embeddings(loc))


# ------------------------------------------------------------------ single-stream layers (a-4, a-5)
class _SelfAttention(nn.Module):
    def __init__(self, hidden, heads):
        super().__init__()
        self.num_attention_heads = heads
        self.attention_head_size = hidden // heads
        self.query = nn.Linear(hidden, hidden)
        self.key = nn.Linear(hidden, hidden)
        self.value = nn.Linear(hidden, hidden)

    def _split(self, x):
        b, l, _ = x.shape
        return x.view(b, l, self.num_attention_heads, self.attention_head_size).permute(0, 2, 1, 3)

    def forward(self, h, ext_mask):
        q, k, v = self._split(self.query(h)), self._split(self.key(h)), self._split(self.value(h))
        s = torch.matmul(q, k.transpose(-1, -2)) / math.sqrt(self.attention_head_size)
        s = s + ext_mask
        p = torch.softmax(s, dim=-1)
        ctx = torch.matmul(p, v).permute(0, 2, 1, 3).contiguous()
        return ctx.view(ctx.size(0), ctx.size(1), -1), p


class _SelfOutput(nn.Module):
    def __init__(self, hidden):
        super().__init__()
        self.dense = nn.Linear(hidden, hidden)
        self.LayerNorm = BertLayerNorm(hidden, eps=1e-12)

    def forward(self, x, residual):
        return self.LayerNorm(self.dense(x) + residual)


class _Attention(nn.Module):
    def __init__(self, hidden, heads):
        super().__init__()
        self.self = _SelfAttention(hidden, heads)
        self.output = _SelfOutput(hidden)

    def forward(self, h, ext_mask):
        ctx, p = self.self(h, ext_mask)
        return self.output(ctx, h), p


class _Intermediate(nn.Module):
    def __init__(self, hidden, inter):
        super().__init__()
        self.dense = nn.Linear(hidden, inter)

    def forward(self, x):
        return gelu(self.dense(x))


class _Output(nn.Module):
    def __init__(self, inter, hidden):
        super().__init__()
        self.dense = nn.Linear(inter, hidden)
        self.LayerNorm = BertLayerNorm(hidden, eps=1e-12)

    def forward(self, x, residual):
        return self.LayerNorm(self.dense(x) + residual)


class BertLayer(nn.Module):
    """Text layer (hidden 768, 12x64 heads, FFN 3072) and, with other sizes, BertImageLayer."""

    def __init__(self, hidden, heads, inter):
        super().__init__()
        self.attention = _Attention(hidden, heads)
        self.intermediate = _Intermediate(hidden, inter)
        self.output = _Output(inter, hidden)

    def forward(self, h, ext_mask):
        a, p = self.attention(h, ext_mask)
        return self.output(self.intermediate(a), a), p


# ------------------------------------------------------------------ co-attention (a-6, a-7)
class BertBiAttention(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.num_attention_heads = c.bi_num_attention_heads
        self.attention_head_size = c.bi_hidden_size // c.bi_num_attention_heads
        hs = c.bi_hidden_size
        self.query1 = nn.Linear(c.v_hidden_size, hs)
        self.key1 = nn.Linear(c.v_hidden_size, hs)
        self.value1 = nn.Linear(c.v_hidden_size, hs)
        self.query2 = nn.Linear(c.hidden_size, hs)
        self.key2 = nn.Linear(c.hidden_size, hs)
        self.value2 = nn.Linear(c.hidden_size, hs)

    def _split(self, x):
        b, l, _ = x.shape
        return x.view(b, l, self.num_attention_heads, self.attention_head_size).permute(0, 2, 1, 3)

    def forward(self, v, v_mask, t, t_mask):
        q1, k1, v1 = self._split(self.query1(v)), self._split(self.key1(v)), self._split(self.value1(v))
        q2, k2, v2 = self._split(self.query2(t)), self._split(self.key2(t)), self._split(self.value2(t))
        d = math.sqrt(self.attention_head_size)
        # text queries over image keys/values -> context for the TEXT stream
        p1 = torch.softmax(torch.matmul(q2, k1.transpose(-1, -2)) / d + v_mask, dim=-1)
        c1 = torch.matmul(p1, v1).permute(0, 2, 1, 3).contiguous()
        c1 = c1.view(c1.size(0), c1.size(1), -1)                      # [B,T,1024]
        # image queries over text keys/values -> context for the IMAGE stream
        p2 = torch.softmax(torch.matmul(q1, k2.transpose(-1, -2)) / d + t_mask, dim=-1)
        c2 = torch.matmul(p2, v2).permute(0, 2, 1, 3).contiguous()
        c2 = c2.view(c2.size(0), c2.size(1), -1)                      # [B,V,1024]
        return c1, c2, (p1, p2)


class BertBiOutput(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.dense1 = nn.Linear(c.bi_hidden_size, c.v_hidden_size)
        self.LayerNorm1 = BertLayerNorm(c.v_hidden_size, eps=1e-12)
        self.q_dense1 = nn.Linear(c.bi_hidden_size, c.v_hidden_size)   # in checkpoint, unused
        self.dense2 = nn.Linear(c.bi_hidden_size, c.hidden_size)
        self.LayerNorm2 = BertLayerNorm(c.hidden_size, eps=1e-12)
        self.q_dense2 = nn.Linear(c.bi_hidden_size, c.hidden_size)     # in checkpoint, unused

    def forward(self, ctx_for_image, v_in, ctx_for_text, t_in):
        v = self.LayerNorm1(self.dense1(ctx_for_image) + v_in)
        t = self.LayerNorm2(self.dense2(ctx_for_text) + t_in)
        return v, t


class BertConnectionLayer(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.biattention = BertBiAttention(c)
        self.biOutput = BertBiOutput(c)
        self.v_intermediate = _Intermediate(c.v_hidden_size, c.v_intermediate_size)
        self.v_output = _Output(c.v_intermediate_size, c.v_hidden_size)
        self.t_intermediate = _Intermediate(c.hidden_size, c.intermediate_size)
        self.t_output = _Output(c.intermediate_size, c.hidden_size)

    def forward(self, v, v_mask, t, t_mask):
        ctx_text, ctx_image, probs = self.biattention(v, v_mask, t, t_mask)
        v_att, t_att = self.biOutput(ctx_image, v, ctx_text, t)
        v_out = self.v_output(self.v_intermediate(v_att), v_att)
        t_out = self.t_output(self.t_intermediate(t_att), t_att)
        return v_out, t_out, probs


class BertEncoder(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.v_biattention_id = list(c.v_biattention_id)
        self.t_biattention_id = list(c.t_biattention_id)
        self.layer = nn.ModuleList([BertLayer(c.hidden_size, c.num_attention_heads, c.intermediate_size)
                                    for _ in range(c.num_hidden_layers)])
        self.v_layer = nn.ModuleList([BertLayer(c.v_hidden_size, c.v_num_attention_heads, c.v_intermediate_size)
                                      for _ in range(c.v_num_hidden_layers)])
        self.c_layer = nn.ModuleList([BertConnectionLayer(c) for _ in range(len(c.v_biattention_id))])

    def schedule(self) -> List[str]:
        """Execution order as strings 'T3' / 'V0' / 'C2' (SURVEY a-8)."""
        order, v_start, t_start = [], 0, 0
        for count, (v_end, t_end) in enumerate(zip(self.v_biattention_id, self.t_biattention_id)):
            order += [f"T{i}" for i in range(t_start, t_end)]
            order += [f"V{i}" for i in range(v_start, v_end)]
            order.append(f"C{count}")
            v_start, t_start = v_end, t_end
        order += [f"V{i}" for i in range(v_start, len(self.v_layer))]
        order += [f"T{i}" for i in range(t_start, len(self.layer))]
        return order

    def forward(self, t, v, t_mask, v_mask, collect=None):
        attn = []
        for step in self.schedule():
            kind, idx = step[0], int(step[1:])
            if kind == "T":
                t, p = self.layer[idx](t, t_mask)
            elif kind == "V":
                v, p = self.v_layer[idx](v, v_mask)
            else:
                v, t, p = self.c_layer[idx](v, v_mask, t, t_mask)
            attn.append(p)
            if collect is not None:
                collect[step] = (t.clone(), v.clone())
        return t, v, attn


class BertTextPooler(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.dense = nn.Linear(c.hidden_size, c.bi_hidden_size)

    def forward(self, h):
        return torch.relu(self.dense(h[:, 0]))


class BertImagePooler(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.dense = nn.Linear(c.v_hidden_size, c.bi_hidden_size)

    def forward(self, h):
        return torch.relu(self.dense(h[:, 0]))


class BertModel(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.task_specific_tokens = c.task_specific_tokens
        self.embeddings = BertEmbeddings(c)
        self.v_embeddings = BertImageEmbeddings(c)
        self.encoder = BertEncoder(c)
        self.t_pooler = BertTextPooler(c)
        self.v_pooler = BertImagePooler(c)

    def forward(self, input_txt, input_imgs, image_loc, token_type_ids, attention_mask,
                image_attention_mask, task_ids, collect=None):
        if self.task_specific_tokens:
            ones = attention_mask.new_ones(attention_mask.size(0), 1)
            attention_mask = torch.cat([ones, attention_mask], dim=1)
        dt = self.embeddings.word_embeddings.weight.dtype              # fp32, or fp64 for an fp64 copy of the oracle
        t_mask = (1.0 - attention_mask[:, None, None, :].to(dt)) * -10000.0
        v_mask = (1.0 - image_attention_mask[:, None, None, :].to(dt)) * -10000.0
        t = self.embeddings(input_txt, token_type_ids, task_ids)
        v = self.v_embeddings(input_imgs, image_loc)
        if collect is not None:
            collect["emb"] = (t.clone(), v.clone())
        t, v, attn = self.encoder(t, v, t_mask, v_mask, collect)
        return t, v, self.t_pooler(t), self.v_pooler(v), attn


# ------------------------------------------------------------------ heads (a-9, a-10)
class _PredictionHeadTransform(nn.Module):
    def __init__(self, hidden):
        super().__init__()
        self.dense = nn.Linear(hidden, hidden)
        self.LayerNorm = BertLayerNorm(hidden, eps=1e-12)

    def forward(self, x):
        return self.LayerNorm(gelu(self.dense(x)))


class BertLMPredictionHead(nn.Module):
    def __init__(self, c, word_embedding_weight):
        super().__init__()
        self.transform = _PredictionHeadTransform(c.hidden_size)
        self.decoder = nn.Linear(c.hidden_size, c.vocab_size, bias=False)
        self.decoder.weight = word_embedding_weight            # tied
        self.bias = nn.Parameter(torch.zeros(c.vocab_size))

    def forward(self, x):
        return self.decoder(self.transform(x)) + self.bias


class BertImagePredictionHead(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.transform = _PredictionHeadTransform(c.v_hidden_size)
        self.decoder = nn.Linear(c.v_hidden_size, c.v_target_size)

    def forward(self, x):
        return self.decoder(self.transform(x))


class BertPreTrainingHeads(nn.Module):
    def __init__(self, c, word_embedding_weight):
        super().__init__()
        self.predictions = BertLMPredictionHead(c, word_embedding_weight)
        self.bi_seq_relationship = nn.Linear(c.bi_hidden_size, 2)
        self.imagePredictions = BertImagePredictionHead(c)

    def forward(self, t, v, pooled_t, pooled_v):
        pooled = pooled_t * pooled_v
        return self.predictions(t), self.imagePredictions(v), self.bi_seq_relationship(pooled)


class SimpleClassifier(nn.Module):
    def __init__(self, in_dim, hid_dim, out_dim):
        super().__init__()
        self.logit_fc = nn.Sequential(nn.Linear(in_dim, hid_dim), GeLU(),
                                      BertLayerNorm(hid_dim, eps=1e-12), nn.Linear(hid_dim, out_dim))

    def forward(self, x):
        return self.logit_fc(x)


class VILBertForVLTasks(nn.Module):
    """Positional forward and 10-tuple of worker.py:287-289."""

    def __init__(self, config: RefConfig, num_labels: int = 3129, gqa_labels: int = 1533):
        super().__init__()
        c = config
        self.config = c
        self.num_labels = num_labels
        self.bert = BertModel(c)
        self.cls = BertPreTrainingHeads(c, self.bert.embeddings.word_embeddings.weight)
        bh = c.bi_hidden_size
        self.vil_prediction = SimpleClassifier(bh, bh * 2, num_labels)
        self.vil_prediction_gqa = SimpleClassifier(bh, bh * 2, gqa_labels)
        self.vil_binary_prediction = SimpleClassifier(bh * 2, bh * 2, 2)
        self.vil_logit = nn.Linear(bh, 1)
        self.vil_tri_prediction = nn.Linear(bh, 3)
        self.vision_logit = nn.Linear(c.v_hidden_size, 1)
        self.linguisic_logit = nn.Linear(c.hidden_size, 1)

    @torch.no_grad()
    def forward(self, input_txt, input_imgs, image_loc, token_type_ids=None, attention_mask=None,
                image_attention_mask=None, co_attention_mask=None, task_ids=None,
                output_all_encoded_layers=False, output_all_attention_masks=False,
                compute_pretraining_heads=True, collect=None):
        if token_type_ids is None:
            token_type_ids = torch.zeros_like(input_txt)
        if attention_mask is None:
            attention_mask = torch.ones_like(input_txt)
        if image_attention_mask is None:
            image_attention_mask = torch.ones(input_imgs.size(0), input_imgs.size(1), dtype=torch.long)
        dt = self.vil_logit.weight.dtype
        t, v, pooled_t, pooled_v, attn = self.bert(input_txt, input_imgs.to(dt), image_loc.to(dt),
                                                   token_type_ids, attention_mask, image_attention_mask,
                                                   task_ids, collect)
        if compute_pretraining_heads:
            linguisic_prediction, vision_prediction, seq_rel = self.cls(t, v, pooled_t, pooled_v)
        else:
            linguisic_prediction = vision_prediction = None
            seq_rel = self.cls.bi_seq_relationship(pooled_t * pooled_v)
        pooled = pooled_t * pooled_v
        vil_prediction = self.vil_prediction(pooled)
        vil_prediction_gqa = self.vil_prediction_gqa(pooled)
        vil_binary_prediction = seq_rel
        if pooled.size(0) % 2 == 0:
            vil_binary_prediction = self.vil_binary_prediction(pooled.view(-1, pooled.size(1) * 2))
        vil_logit = self.vil_logit(pooled)
        vil_tri_prediction = self.vil_tri_prediction(pooled)
        vision_logit = self.vision_logit(v) + ((1.0 - image_attention_mask.to(dt)) * -10000.0).unsqueeze(2)
        linguisic_logit = self.linguisic_logit(t)
        if collect is not None:
            collect["final"] = (t, v, pooled_t, pooled_v)
        return (vil_prediction, vil_prediction_gqa, vil_logit, vil_binary_prediction, vil_tri_prediction,
                vision_prediction, vision_logit, linguisic_prediction, linguisic_logit,
                attn if output_all_attention_masks else [])


# ------------------------------------------------------------------ utilities
def count_parameters(model: nn.Module) -> int:
    seen, n = set(), 0
    for p in model.parameters():
        if id(p) not in seen:
            seen.add(id(p))
            n += p.numel()
    return n


def init_weights(model: nn.Module, seed: int = 42, logit_gain: float = 10.0, bf16_exact: bool = True):
    """Seeded synthetic weights (SURVEY.md section 8d-1; seed echoes worker.py:477).

    Linear/Embedding ~ N(0, 0.02); LN gamma ~ 1 + N(0, 0.1), beta ~ N(0, 0.1); biases ~ N(0, 0.05);
    plain-Linear head layers x logit_gain so every logit family has O(1) spread (otherwise those logits
    are ~0 and an absolute tolerance is vacuous).  With ``bf16_exact`` the Linear weights are rounded to
    bf16-representable values, i.e. the synthetic checkpoint is one that bf16 storage reproduces
    exactly, so oracle (fp32 math) and engine (bf16 operands) start from identical parameters.
    """
    g = torch.Generator().manual_seed(seed)
    # plain-Linear heads read small pooled/hidden values -> x logit_gain; the SimpleClassifier output layers
    # already see a unit-variance LayerNorm output over 2048 dims (std ~ sqrt(2048)*0.02 ~ 0.9) -> gain 1.
    out_layers = {"vil_logit", "vil_tri_prediction", "vision_logit", "linguisic_logit", "cls.bi_seq_relationship"}
    with torch.no_grad():
        for name, m in model.named_modules():
            if isinstance(m, nn.Linear):
                m.weight.copy_(torch.randn(m.weight.shape, generator=g) * 0.02)
                if name in out_layers:
                    m.weight.mul_(logit_gain)
                if bf16_exact:
                    m.weight.copy_(m.weight.to(torch.bfloat16).float())
                if m.bias is not None:
                    m.bias.copy_(torch.randn(m.bias.shape, generator=g) * 0.05)
            elif isinstance(m, nn.Embedding):
                m.weight.copy_(torch.randn(m.weight.shape, generator=g) * 0.02)
            elif isinstance(m, BertLayerNorm):
                m.weight.copy_(1.0 + torch.randn(m.weight.shape, generator=g) * 0.1)
                m.bias.copy_(torch.randn(m.bias.shape, generator=g) * 0.1)
        model.cls.predictions.bias.copy_(torch.randn(model.cls.predictions.bias.shape, generator=g) * 0.05)
    return model


def make_inputs(batch: int, n_tokens: int = 30, n_regions: int = 36, seed: int = 1234, task_id: int = 1,
                full_masks: bool = False, vocab_size: int = 30522, pad_regions: int = 0):
    """Synthetic request tensors in the shapes/dtypes of worker.py:416-419, 452-455 (SURVEY 8d-1).

    features = relu(N(0,1))*1.5 with row 0 the mean of the others (worker.py:432-434); spatials are
    normalised boxes with row 0 = [0,0,1,1,1] (worker.py:443); question = [CLS] ids [SEP] pad...;
    ``pad_regions`` > 0 masks that many trailing regions (image_mask = 0) to exercise the mask path.
    """
    g = torch.Generator().manual_seed(seed)
    B, L, V = batch, n_tokens, n_regions
    feats = torch.relu(torch.randn(B, V, 2048, generator=g)) * 1.5
    if V > 1:
        feats[:, 0] = feats[:, 1:].mean(dim=1)
    x1 = torch.rand(B, V, generator=g) * 0.7
    y1 = torch.rand(B, V, generator=g) * 0.7
    w = 0.05 + torch.rand(B, V, generator=g) * 0.25
    h = 0.05 + torch.rand(B, V, generator=g) * 0.25
    x2, y2 = (x1 + w).clamp(max=1.0), (y1 + h).clamp(max=1.0)
    spatials = torch.stack([x1, y1, x2, y2, (x2 - x1) * (y2 - y1)], dim=-1)
    spatials[:, 0] = torch.tensor([0.0, 0.0, 1.0, 1.0, 1.0])
    question = torch.zeros(B, L, dtype=torch.long)
    input_mask = torch.zeros(B, L, dtype=torch.long)
    for b in range(B):
        n = L - 2 if full_masks else int(torch.randint(min(5, L - 2), max(min(5, L - 2) + 1, L - 1), (1,), generator=g))
        n = max(1, min(n, L - 2))
        ids = torch.randint(1000, vocab_size, (n,), generator=g)
        question[b, 0] = 101
        question[b, 1:1 + n] = ids
        question[b, 1 + n] = 102
        input_mask[b, :n + 2] = 1
    segment_ids = torch.zeros(B, L, dtype=torch.long)
    image_mask = torch.ones(B, V, dtype=torch.uint8)
    if pad_regions > 0:
        image_mask[:, V - pad_regions:] = 0
    co_attention_mask = torch.zeros(B, V, L)
    task_tokens = torch.full((B, 1), task_id, dtype=torch.long)
    return question, feats, spatials, segment_ids, input_mask, image_mask, co_attention_mask, task_tokens


def build(config: Optional[RefConfig] = None, seed: int = 42, num_labels: int = 3129) -> VILBertForVLTasks:
    model = VILBertForVLTasks(config or RefConfig(), num_labels=num_labels)
    init_weights(model, seed=seed)
    return model.eval()


class emulate_activation_rounding:
    """Context manager: run the oracle with the engine's 16-bit activation rounding points, everything else fp32.

    The engine rounds (to fp16 or bf16) exactly the operands it feeds to tensor-core GEMMs -- the input of every
    wide nn.Linear, the 5-d box operand of the image embedding included -- and the Q/K/V projections it hands to the
    attention kernels.  The narrow heads (vil_logit, vil_tri_prediction, vision_logit, linguisic_logit,
    bi_seq_relationship and the 2-wide last layer of vil_binary_prediction) read fp32.  With this emulation the
    oracle becomes "what exact 16-bit arithmetic gives", so engine-vs-emulation isolates kernel bugs from the
    unavoidable rounding of the chosen activation format.
    """
    NARROW = ("vil_logit", "vil_tri_prediction", "vision_logit", "linguisic_logit", "cls.bi_seq_relationship",
              "vil_binary_prediction.logit_fc.3")
    QKV = ("query", "key", "value", "query1", "key1", "value1", "query2", "key2", "value2")

    def __init__(self, model: nn.Module, dtype: torch.dtype):
        self.model, self.dtype, self.hooks = model, dtype, []

    def __enter__(self):
        dt = self.dtype

        def pre(_mod, args):
            return (args[0].to(dt).float(),)

        def post(_mod, _args, out):
            return out.to(dt).float()
        for name, mod in self.model.named_modules():
            if isinstance(mod, nn.Linear) and name not in self.NARROW:
                self.hooks.append(mod.register_forward_pre_hook(pre))
                if name.rsplit(".", 1)[-1] in self.QKV:
                    self.hooks.append(mod.register_forward_hook(post))
        return self

    def __exit__(self, *exc):
        for h in self.hooks:
            h.remove()
        return False


def tiny_config(**kw) -> RefConfig:
    """A structurally identical but small model (same 12/6/6 schedule) for second-scale CPU tests."""
    d = dict(hidden_size=128, num_attention_heads=2, intermediate_size=256,
             v_hidden_size=256, v_num_attention_heads=2, v_intermediate_size=256,
             bi_hidden_size=256, bi_num_attention_heads=2, bi_intermediate_size=256,
             vocab_size=2048, v_feature_size=256, v_target_size=64, max_position_embeddings=160)
    d.update(kw)
    return RefConfig(**d)
