"""CPU/torch oracle (test infrastructure) of HF RobertaModel's forward, built on `oracle.bert_oracle`.

RobertaModel is BertModel with two differences in its embeddings (transformers 5.5 modeling_roberta.py):
  - positions: `create_position_ids_from_input_ids` = padding_idx + cumsum(id != padding_idx) for a non-pad id and
    padding_idx for a pad id, over the whole (padded) row, so a pad id inside the text is not counted;
  - a token-type table of type_vocab_size rows (1 for roberta-base), indexed by zeros when token_type_ids is None.
The layers are BERT's.  `bert_oracle.bert_hidden` runs one sequence at a time on its real tokens with the position
table gathered at that sequence's RoBERTa positions (its own position rule is row t for token t), which is the same
arithmetic as HF's padded batch for every real token."""
from typing import Dict

import torch

from oracle import bert_oracle as BO


def roberta_positions(input_ids: torch.Tensor, padding_idx: int = 1) -> torch.Tensor:
    """HF `create_position_ids_from_input_ids` on [B, S] (or [S]) ids."""
    mask = input_ids.ne(padding_idx).long()
    return torch.cumsum(mask, dim=-1) * mask + padding_idx


def roberta_token_rows(sd: Dict[str, torch.Tensor], config: dict, input_ids, attention_mask, dtype=torch.float32,
                       padding_idx: int = 1) -> torch.Tensor:
    """last_hidden_state rows of the real tokens (attention_mask == 1), in batch order: [T, hidden] in `dtype`."""
    pos_table = sd["embeddings.position_embeddings.weight"]
    pos = roberta_positions(input_ids, padding_idx)
    rows = []
    for b in range(input_ids.shape[0]):
        m = attention_mask[b].bool()
        ids = input_ids[b][m][None]
        if ids.shape[1] == 0:
            continue
        p = pos[b][m].to(pos_table.device)
        if int(p.max()) >= pos_table.shape[0]:
            raise IndexError(f"sequence {b}: position {int(p.max())} is past max_position_embeddings")
        sd_b = dict(sd)
        sd_b["embeddings.position_embeddings.weight"] = pos_table[p]
        rows.append(BO.bert_hidden(sd_b, config, ids, torch.ones_like(ids), None, dtype)[0])
    return torch.cat(rows)


def roberta_cls(sd, config, input_ids, attention_mask, dtype=torch.float32, padding_idx: int = 1) -> torch.Tensor:
    """`last_hidden_state[:, 0, :]` (the reference's CLS branch, src/search.py:93-94): [B, hidden]."""
    rows = roberta_token_rows(sd, config, input_ids, attention_mask, dtype, padding_idx)
    lens = attention_mask.sum(dim=1).long().cpu()
    starts = torch.cumsum(lens, 0) - lens
    return rows[starts.to(rows.device)]
