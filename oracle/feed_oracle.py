"""Restatement of the reference training dataset (BaseDataset, src/dataset.py:17-85): one item per behaviour row, built on
the host, in the format default_collate turns into the trainer's minibatch.  It is the baseline of tools/feed_bench.py
and is checked against batches collated from the reference itself (tests/golden/feed.npz).

Item of row r: "clicked" the labels of its candidates; "candidate_news" one dict {attribute: tensor} per candidate;
"clicked_news" the first num_clicked_news_a_user browsed news, preceded by as many all-zero padding news as make up the
difference; "user" and "clicked_news_length" (the history length after truncation) when the config's record list has them.
Category and subcategory are 0-d tensors, the list attributes 1-d.
"""
from __future__ import annotations

from ast import literal_eval

import torch
from torch.utils.data import Dataset

LIST_ATTRIBUTES = ("title", "abstract", "title_entities", "abstract_entities")


class FeedOracle(Dataset):
    def __init__(self, behaviors_path, news_path, config):
        import pandas as pd
        self.H = int(config.num_clicked_news_a_user)
        self.attributes = list(config.dataset_attributes["news"])
        self.records = list(config.dataset_attributes["record"])
        self.rows = pd.read_table(behaviors_path)
        table = pd.read_table(news_path, usecols=["id"] + self.attributes,
                              converters={a: literal_eval for a in self.attributes if a in LIST_ATTRIBUTES})
        self.news = {}
        for rec in table.to_dict("records"):
            key = rec.pop("id")
            self.news[key] = {a: torch.tensor(v) for a, v in rec.items()}
        width = {"title": config.num_words_title, "title_entities": config.num_words_title,
                 "abstract": config.num_words_abstract, "abstract_entities": config.num_words_abstract}
        self.padding = {a: torch.zeros(width[a], dtype=torch.int64) if a in width else torch.tensor(0) for a in self.attributes}

    def __len__(self):
        return len(self.rows)

    def __getitem__(self, idx):
        row = self.rows.iloc[idx]
        history = [self.news[x] for x in row["clicked_news"].split()[:self.H]]
        item = {"clicked": [int(x) for x in row["clicked"].split()],
                "candidate_news": [self.news[x] for x in row["candidate_news"].split()],
                "clicked_news": [self.padding] * (self.H - len(history)) + history}
        if "user" in self.records:
            item["user"] = int(row["user"])
        if "clicked_news_length" in self.records:
            item["clicked_news_length"] = len(history)
        return item
