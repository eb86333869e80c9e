"""Text-encoder wrapper on the caller side of the hot path (reference: modeling/modeling_encoder.py:89-143).

Out of scope for the CUDA kernels ("drops in behind the existing RoBERTa encoder"): this is a thin
HuggingFace wrapper with the reference's interface — `TextEncoder(model_name, **kwargs)`, `.sent_dim`,
`forward(input_ids, attention_mask, token_type_ids, output_mask, layer_id=-1) -> (sent_vecs, all_hidden_states)`
— for the BERT/RoBERTa family the QA-GNN configs use.  Offline environments pass
`config=<PretrainedConfig>` (random init) instead of downloading a checkpoint.
"""
import torch.nn as nn


class TextEncoder(nn.Module):
    def __init__(self, model_name, output_token_states=False, from_checkpoint=None, config=None, **kwargs):
        super().__init__()
        from transformers import AutoModel
        self.output_token_states = output_token_states
        if config is not None:
            config.output_hidden_states = True
            self.module = AutoModel.from_config(config)
        else:
            self.module = AutoModel.from_pretrained(from_checkpoint or model_name, output_hidden_states=True)
        self.model_type = self.module.config.model_type
        if self.model_type not in ("bert", "roberta", "albert", "xlm-roberta"):
            raise NotImplementedError(f"TextEncoder: model type {self.model_type!r} is outside the QA-GNN configs")
        self.sent_dim = self.module.config.hidden_size

    def forward(self, *inputs, layer_id=-1):
        input_ids, attention_mask, token_type_ids, output_mask = inputs
        outputs = self.module(input_ids, token_type_ids=token_type_ids, attention_mask=attention_mask,
                              output_hidden_states=True)
        all_hidden_states = outputs.hidden_states
        hidden_states = all_hidden_states[layer_id]
        if self.output_token_states:
            return hidden_states, output_mask
        if self.model_type == "albert":
            return hidden_states[:, 0], all_hidden_states
        return self.module.pooler(hidden_states), all_hidden_states
