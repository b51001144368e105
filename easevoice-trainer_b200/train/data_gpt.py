"""Stage-1 input side: dataset over `2-name2text.txt` + `6-name2semantic.tsv` (+ `3-bert/<name>.pt`), pad-collate and the
duration-bucketed distributed sampler.  Reference: src/easevoice/soundstorm/auto_reg/data/dataset.py:40-271,
bucket_sampler.py:30-167, data_module.py:39-53.  Same filtering rules, same batch dict
(`phoneme_ids, phoneme_ids_len, semantic_ids (pad 1024), semantic_ids_len, bert_feature [B, 1024, Xmax]`)."""
import itertools
import math
import os
import random

import numpy as np
import torch


class Text2SemanticDataset(torch.utils.data.Dataset):
    def __init__(self, phoneme_path, semantic_path, max_sample=None, max_sec=100, pad_val=1024, min_ps_ratio=3, max_ps_ratio=25,
                 phoneme_table=None, hz=25):
        assert os.path.exists(phoneme_path), phoneme_path
        assert os.path.exists(semantic_path), semantic_path
        if phoneme_table is None:
            from .data import default_phoneme_table
            phoneme_table = default_phoneme_table()
        self.path3 = os.path.join(os.path.dirname(phoneme_path), "3-bert")
        self.PAD, self.hz = pad_val, hz
        phon = {}
        with open(phoneme_path, encoding="utf8") as f:
            for line in f.read().strip("\n").split("\n"):
                t = line.split("\t")
                if len(t) == 4:
                    phon[t[0]] = t[1]
        rows = []
        with open(semantic_path, encoding="utf-8") as f:
            lines = f.read().strip("\n").split("\n")
        for line in lines[1:]:                                     # pandas.read_csv consumes the first line as the header
            t = line.split("\t")
            if len(t) >= 2:
                rows.append((t[0], t[1]))
        if max_sample is not None:
            rows = rows[:max_sample]
        self.semantic_phoneme, self.item_names = [], []
        for name, sem in rows:
            if name not in phon:
                continue
            semantic_ids = [int(i) for i in sem.split(" ")]
            if len(semantic_ids) > max_sec * hz:
                continue
            try:
                phoneme_ids = [phoneme_table[p] for p in phon[name].split(" ")]
            except KeyError:
                continue
            if len(phoneme_ids) > max_sec * hz / 2.5:
                continue
            ps = len(phoneme_ids) / (len(semantic_ids) / hz)
            if ps > max_ps_ratio or ps < min_ps_ratio:
                continue
            self.semantic_phoneme.append((semantic_ids, phoneme_ids))
            self.item_names.append(name)
        n = len(self.semantic_phoneme)
        if n == 0:
            raise ValueError(f"no valid data in {semantic_path}, please check the data and try again")
        if n < 100:                                                # dataset.py:150-158: tiny sets are replicated
            rep = max(2, int(100 / n))
            self.semantic_phoneme, self.item_names = self.semantic_phoneme * rep, self.item_names * rep

    def __len__(self):
        return len(self.semantic_phoneme)

    def get_sample_length(self, idx):
        return 1.0 * len(self.semantic_phoneme[idx][0]) / self.hz

    def __getitem__(self, idx):
        semantic_ids, phoneme_ids = self.semantic_phoneme[idx]
        path_bert = os.path.join(self.path3, f"{self.item_names[idx]}.pt")
        bert = None
        if os.path.exists(path_bert):
            bert = torch.load(path_bert, map_location="cpu")
            assert bert.shape[-1] == len(phoneme_ids)
        return dict(idx=idx, phoneme_ids=phoneme_ids, phoneme_ids_len=len(phoneme_ids), semantic_ids=semantic_ids,
                    semantic_ids_len=len(semantic_ids), bert_feature=bert)

    def collate(self, examples):
        B = len(examples)
        xl = torch.tensor([e["phoneme_ids_len"] for e in examples], dtype=torch.int64)
        yl = torch.tensor([e["semantic_ids_len"] for e in examples], dtype=torch.int64)
        x = torch.zeros((B, int(xl.max())), dtype=torch.int64)
        y = torch.full((B, int(yl.max())), self.PAD, dtype=torch.int64)
        bert = torch.zeros((B, 1024, int(xl.max())), dtype=torch.float32)
        for i, e in enumerate(examples):
            x[i, :xl[i]] = torch.as_tensor(np.asarray(e["phoneme_ids"], dtype=np.int64))
            y[i, :yl[i]] = torch.as_tensor(np.asarray(e["semantic_ids"], dtype=np.int64))
            if e["bert_feature"] is not None:
                bert[i, :, :e["bert_feature"].shape[-1]] = e["bert_feature"]
        return dict(ids=[e["idx"] for e in examples], phoneme_ids=x, phoneme_ids_len=xl, semantic_ids=y, semantic_ids_len=yl,
                    bert_feature=bert)


def pad_host_batch(host, Xq, Yq, pad_val=1024):
    """Pad a collated batch (Text2SemanticDataset.collate layout) to Xq phonemes / Yq semantic tokens: phonemes and BERT
    features with 0, semantic ids with pad_val, as the collate pads.  The lengths are unchanged, so the padding is inert
    apart from the loss terms the counted length removes (GptStep.prepare).  Pinned inputs give pinned outputs, so the
    copies to the device stay asynchronous."""
    B, X = host["phoneme_ids"].shape
    Y = host["semantic_ids"].shape[1]
    if X == Xq and Y == Yq:
        return host
    assert Xq >= X and Yq >= Y
    pin = host["semantic_ids"].is_pinned()
    out = dict(host)
    for k, shape, fill in (("phoneme_ids", (B, Xq), 0), ("semantic_ids", (B, Yq), pad_val), ("bert_feature", (B, 1024, Xq), 0)):
        src = host[k]
        dst = torch.full(shape, fill, dtype=src.dtype, pin_memory=pin)
        dst[..., :src.shape[-1]] = src
        out[k] = dst
    return out


class DistributedBucketSampler(torch.utils.data.Sampler):
    """bucket_sampler.py:30-167: 2-second duration buckets, shuffle inside buckets, chunk into world*batch groups, shuffle
    the groups, pad to a multiple of world, stride by rank.  Yields sample indices (the DataLoader batches them)."""

    def __init__(self, dataset, num_replicas=1, rank=0, shuffle=True, seed=0, batch_size=32):
        self.dataset, self.num_replicas, self.rank, self.shuffle, self.seed, self.batch_size = dataset, num_replicas, rank, shuffle, seed, batch_size
        self.epoch = 0
        self.num_samples = math.ceil(len(dataset) / num_replicas)
        self.total_size = self.num_samples * num_replicas
        ids = sorted(((i, dataset.get_sample_length(i)) for i in range(len(dataset))), key=lambda t: t[1])
        self.id_buckets, cur, max_sec = [], [], 2.0
        for i, sec in ids:
            if sec < max_sec:
                cur.append(i)
            else:
                self.id_buckets.append(cur)
                cur = [i]
                max_sec += 2.0
        if cur:
            self.id_buckets.append(cur)

    def __iter__(self):
        if self.shuffle:
            rnd = random.Random(self.epoch + self.seed)
            flat = []
            for buc in self.id_buckets:
                b = list(buc)
                rnd.shuffle(b)
                flat += b
            gb = self.batch_size * self.num_replicas
            batches = [flat[i * gb:(i + 1) * gb] for i in range(int(math.ceil(len(flat) / gb)))]
            rnd.shuffle(batches)
            indices = list(itertools.chain(*batches))
        else:
            indices = list(range(len(self.dataset)))
        pad = self.total_size - len(indices)
        if pad <= len(indices):
            indices += indices[:pad]
        else:
            indices += (indices * math.ceil(pad / len(indices)))[:pad]
        return iter(indices[self.rank:self.total_size:self.num_replicas])

    def __len__(self):
        return self.num_samples

    def set_epoch(self, epoch):
        self.epoch = epoch
