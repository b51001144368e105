"""Stage-1 trainer with the reference's class API (src/train/gpt.py:27-39, 93-177):
    GPTTrainParams(...)  ->  GPTTrain(params).train() -> TrainOutput(model_path)
Same parameter dataclass (field names are the REST wire format), same configs/gpt.yaml schema, same directory scheme
(<project_dir>/models/gpt_train/<name>/{logs/ckpt/epoch=E-step=S.ckpt, <name>-e{E}.ckpt}), same stdout protocol
(`loss-of-easevoice {"step","loss","acc","lr","epoch"}` every step on rank 0, t2s_lightning_module.py:83-89).
The Lightning Trainer/DDPStrategy/ModelCheckpoint machinery is replaced by a plain loop around train/gpt_step.GptStep; the
checkpoint files keep Lightning's keys ("state_dict" with the "model." prefix, "epoch", "global_step",
"optimizer_states") so `_get_newest_ckpt` style resume and the reference's weight loaders keep working."""
import os
import re
from collections import OrderedDict
from dataclasses import dataclass
from random import randint

import torch
import torch.distributed as dist
import yaml

from .. import ops
from ..models_gpt import Text2SemanticDecoder
from ..utils.connector import MultiProcessOutputConnector
from . import data_gpt, gpt_step
from .helper import TrainOutput, get_gpt_train_dir, train_logs_path

GPT_PRETRAINED = "pretrained/gsv-v2final-pretrained/s1bert25hz-5kh-longer-epoch=12-step=369668.ckpt"
HERE = os.path.dirname(os.path.abspath(__file__))
GPT_CONFIG_PATH = os.path.join(os.path.dirname(os.path.dirname(HERE)), "configs", "gpt.yaml")


@dataclass
class GPTTrainParams:
    batch_size: int = 12
    total_epochs: int = 15
    save_every_epoch: int = 5
    if_dpo: bool = False
    if_save_latest: bool = True
    if_save_every_weights: bool = True
    gpu_ids: str = "0"
    model_path: str = GPT_PRETRAINED
    train_input_dir: str = ""
    output_model_name: str = ""
    project_dir: str = ""


class GPTTrain:
    def __init__(self, params: GPTTrainParams, dataset=None, config_path=GPT_CONFIG_PATH):
        with open(config_path) as f:
            self.config = yaml.safe_load(f)
        c, t = self.config, self.config["train"]
        self.params, self.dataset = params, dataset
        self.train_output = get_gpt_train_dir(params.project_dir, params.output_model_name)
        self.train_logs_output = os.path.join(self.train_output, train_logs_path)
        self.train_ckpts_output = os.path.join(self.train_logs_output, "ckpt")
        os.makedirs(self.train_ckpts_output, exist_ok=True)
        t["precision"] = "tf32"                       # fp32 storage + TF32 tensor-core math (no autocast / GradScaler)
        t["batch_size"], t["epochs"], t["save_every_n_epoch"] = params.batch_size, params.total_epochs, params.save_every_epoch
        t["if_dpo"], t["if_save_latest"], t["if_save_every_weights"] = params.if_dpo, params.if_save_latest, params.if_save_every_weights
        t["half_weights_save_dir"], t["output_name"] = self.train_output, params.output_model_name
        c["pretrained_s1"] = params.model_path
        c["train_semantic_path"] = os.path.join(params.train_input_dir, "6-name2semantic.tsv")
        c["train_phoneme_path"] = os.path.join(params.train_input_dir, "2-name2text.txt")
        c["logs_output_dir"] = self.train_logs_output
        self.global_step = 0                          # Lightning's global_step counts optimizer steps

    def train(self):
        gpus = [g for g in self.params.gpu_ids.replace("-", ",").split(",") if g != ""]
        if len(gpus) <= 1 or "RANK" in os.environ:
            self._run(int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1)),
                      int(os.environ.get("LOCAL_RANK", gpus[0] if gpus else 0)))
        else:
            import torch.multiprocessing as mp
            os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
            os.environ.setdefault("MASTER_PORT", str(randint(30000, 55555)))
            mp.spawn(_spawn_entry, nprocs=len(gpus), args=(len(gpus), self.params, [int(g) for g in gpus]))
        return TrainOutput(model_path=self.train_output)

    # --------------------------------------------------------------------------------------------
    @staticmethod
    def _get_newest_ckpt(file_list):
        best = None
        for s in file_list or []:
            m = re.match(r"epoch=(\d+)-step=(\d+)\.ckpt", s)
            if m and (best is None or (int(m.group(1)), int(m.group(2))) > best[:2]):
                best = (int(m.group(1)), int(m.group(2)), s)
        return best[2] if best else None

    def _build(self, device):
        torch.manual_seed(self.config["train"]["seed"])
        net = Text2SemanticDecoder(self.config, top_k=3)
        path = self.config.get("pretrained_s1")
        if path and os.path.exists(path):             # t2s_lightning_module.py:25-31 (keys carry the "model." prefix)
            w = torch.load(path, map_location="cpu")["weight"]
            net.load_state_dict({k[len("model."):]: v.float() for k, v in w.items() if k.startswith("model.")})
        return net.to(device).train()

    def _run(self, rank, world, local_rank):
        c, t = self.config, self.config["train"]
        device = torch.device("cuda", local_rank)
        torch.cuda.set_device(device)
        if world > 1 and not dist.is_initialized():
            dist.init_process_group("nccl", rank=rank, world_size=world, device_id=device)
        net = self._build(device)
        step = self.gpt_step = gpt_step.GptStep(net, world_size=world, dpo=bool(t["if_dpo"]))
        ops.manual_seed(t["seed"] + rank)
        ds = self.dataset or data_gpt.Text2SemanticDataset(c["train_phoneme_path"], c["train_semantic_path"],
                                                            max_sec=c["data"]["max_sec"], pad_val=c["data"]["pad_val"])
        bs = t["batch_size"] // 2 if t["if_dpo"] else t["batch_size"]           # data_module.py:39-41
        bs = max(min(bs, len(ds) // 4), 1)
        sampler = data_gpt.DistributedBucketSampler(ds, world, rank, batch_size=bs)
        # two worker processes: in the main process, loading and collating (~20 ms per batch of 12) stalled the GPU step
        # (tools/bench_gpt_train.py); the sampler order and the main process's RNG draws are the same
        loader = torch.utils.data.DataLoader(ds, batch_size=bs, sampler=sampler, collate_fn=ds.collate, num_workers=2, pin_memory=True)
        start_epoch = 0
        newest = self._get_newest_ckpt(os.listdir(self.train_ckpts_output))
        if newest:                                    # resume (gpt.py:171-172)
            sd = torch.load(os.path.join(self.train_ckpts_output, newest), map_location="cpu")
            net.load_state_dict({k[len("model."):]: v.float() for k, v in sd["state_dict"].items()})
            step.opt.load_state_dict(sd["optimizer_states"][0])
            start_epoch, self.global_step = sd["epoch"] + 1, sd["global_step"]
        connector = MultiProcessOutputConnector()
        cstep = 0
        for epoch in range(start_epoch, t["epochs"]):
            sampler.set_epoch(epoch)
            step.batch_idx = 0                        # Lightning's batch_idx restarts every epoch; grads carry over
            for host in loader:
                # padded to the agreed 32-token grid; the loss still counts the collate's shape only (GptStep.prepare)
                batch = step.prepare(host, device)
                did = step.wants_step()
                loss, acc = step.train_step(batch)
                self.global_step += int(did)
                if rank == 0:                         # the only host reads of the loop (t2s_lightning_module.py:83-89)
                    connector.write_loss(cstep, loss=float(loss), other={"acc": float(acc), "lr": step.lr, "epoch": epoch})
                    cstep += 1
            if rank == 0 and (epoch + 1) % t["save_every_n_epoch"] == 0:
                self._save(epoch, net, step)
        if world > 1:
            dist.barrier()

    def _save(self, epoch, net, step):
        t = self.config["train"]
        if t["if_save_latest"]:                       # gpt.py:66-77: keep only the newest trainer checkpoint
            for n in os.listdir(self.train_ckpts_output):
                try:
                    os.remove(os.path.join(self.train_ckpts_output, n))
                except OSError:
                    pass
        sd = OrderedDict(("model." + k, v.detach().cpu().clone()) for k, v in net.state_dict().items())
        torch.save(dict(epoch=epoch, global_step=self.global_step, state_dict=sd, optimizer_states=[step.opt.state_dict()],
                        lr_schedulers=[dict(lr=step.lr)], hyper_parameters=dict(config=self.config)),
                   os.path.join(self.train_ckpts_output, f"epoch={epoch}-step={self.global_step}.ckpt"))
        if t["if_save_every_weights"]:                # gpt.py:78-90: fp16 export consumed by TTS.init_t2s_weights
            od = OrderedDict(weight=OrderedDict((k, v.half()) for k, v in sd.items()), config=self.config, info=f"GPT-e{epoch + 1}")
            torch.save(od, os.path.join(t["half_weights_save_dir"], f"{t['output_name']}-e{epoch + 1}.ckpt"))


def _spawn_entry(local_rank, world, params, gpu_ids):
    os.environ.update(RANK=str(local_rank), WORLD_SIZE=str(world), LOCAL_RANK=str(gpu_ids[local_rank]))
    GPTTrain(params).train()
