"""Stage-2 trainer with the reference's class API (src/train/sovits.py:37-50, 128-211):

    SovitsTrain(SovitsTrainParams(...)).train() -> TrainOutput(model_path)

Same parameter dataclass (field names are the REST wire format), same config file (configs/s2.json), same output
directory scheme, checkpoint/export layouts and stdout progress protocol.  The training loop itself runs on the
sm_90a kernels (S2Step, CUDA-graph replay per batch shape) and is data-parallel over `gpu_ids` with NCCL:
one process per GPU (the reference hard-codes n_gpus = 1, sovits.py:199-210).
"""
import logging
import os
from dataclasses import dataclass
from random import randint

import torch
import torch.distributed as dist

from .. import configs, models, ops
from ..utils import ckpt
from ..utils.connector import MultiProcessOutputConnector
from . import data as s2data
from . import s2_step
from .s2_step import pad_host_batch as s2data_pad
from .helper import TrainOutput, get_sovits_train_dir, train_logs_path

logger = logging.getLogger("easevoice_b200")


def base_path():
    """The host application's root (reference: src/utils/path/path.py:16-19; trainers are started with cwd = base_path,
    session.py:234-253).  Pretrained weights and TensorBoard event files are resolved against it."""
    return os.environ.get("EASEVOICE_BASE_PATH", os.getcwd())


def default_pretrained_s2g():
    """src/utils/config/__init__.py:35"""
    return os.path.join(base_path(), "models", "pretrained", "gsv-v2final-pretrained", "s2G2333k.pth")


def tensorboard_log_dir(name):
    """src/service/tensorboard.py:11-24 (tb_log_dir = <base_path>/tb_logs)."""
    root = os.path.join(base_path(), "tb_logs")
    return root if name is None else os.path.join(root, name)
BUCKET_BOUNDARIES = [32, 300, 400, 500, 600, 700, 800, 900, 1000, 1100, 1200, 1300, 1400, 1500, 1600, 1700, 1800, 1900]


@dataclass
class SovitsTrainParams:
    batch_size: int = 12
    total_epochs: int = 8
    text_low_lr_rate: float = 0.4
    pretrained_s2G: str = ""
    pretrained_s2D: str = ""
    if_save_latest: bool = True
    if_save_every_weights: bool = True
    save_every_epoch: int = 5
    gpu_ids: str = "0"
    train_input_dir: str = ""
    output_model_name: str = ""
    project_dir: str = ""


class SovitsTrain:
    def __init__(self, params: SovitsTrainParams, dataset=None):
        hps = configs.load_s2_config()
        t = hps["train"]
        t["batch_size"], t["epochs"], t["text_low_lr_rate"] = params.batch_size, params.total_epochs, params.text_low_lr_rate
        t["if_save_latest"], t["if_save_every_weights"] = params.if_save_latest, params.if_save_every_weights
        t["save_every_epoch"], t["gpu_numbers"] = params.save_every_epoch, params.gpu_ids
        # sovits.py:148-157: an empty / stock value resolves to the application's default pretrained checkpoints
        g_def = default_pretrained_s2g()
        stock = "pretrained/gsv-v2final-pretrained/s2%s2333k.pth"
        t["pretrained_s2G"] = g_def if params.pretrained_s2G in ("", stock % "G") else params.pretrained_s2G
        t["pretrained_s2D"] = g_def.replace("s2G", "s2D") if params.pretrained_s2D in ("", stock % "D") else params.pretrained_s2D
        hps["name"] = params.output_model_name
        hps["data"]["exp_dir"] = params.train_input_dir
        t["output_dir"] = get_sovits_train_dir(params.project_dir, params.output_model_name)
        t["train_logs_dir"] = os.path.join(t["output_dir"], train_logs_path)
        t["save_weight_dir"] = t["output_dir"]
        os.makedirs(t["train_logs_dir"], exist_ok=True)
        self.hps, self.params, self.dataset = hps, params, dataset
        self.global_step = 0

    # --------------------------------------------------------------------------------------------
    def train(self):
        gpus = [g for g in self.hps["train"]["gpu_numbers"].replace("-", ",").split(",") if g != ""]
        if len(gpus) <= 1 or "RANK" in os.environ:
            rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
            self._run(rank, world, int(os.environ.get("LOCAL_RANK", gpus[0] if gpus else 0)))
        else:
            import torch.multiprocessing as mp
            os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
            os.environ.setdefault("MASTER_PORT", str(randint(30000, 55555)))
            mp.spawn(_spawn_entry, nprocs=len(gpus), args=(len(gpus), self.params, [int(g) for g in gpus], self.dataset))
        return TrainOutput(model_path=self.hps["train"]["output_dir"])

    def _build(self, device):
        hps = self.hps
        torch.manual_seed(hps["train"]["seed"])
        net_g = models.SynthesizerTrn(hps["data"]["filter_length"] // 2 + 1,
                                      hps["train"]["segment_size"] // hps["data"]["hop_length"],
                                      n_speakers=hps["data"]["n_speakers"], **hps["model"])
        net_d = models.MultiPeriodDiscriminator(hps["model"]["use_spectral_norm"])
        return net_g.to(device).train(), net_d.to(device).train()

    def _load_pretrained(self, net_g, net_d):
        """sovits.py:345-366: only when no resumable checkpoint was found."""
        t = self.hps["train"]
        for path, net, strict in ((t["pretrained_s2G"], net_g, False), (t["pretrained_s2D"], net_d, True)):
            if path and os.path.exists(path):
                sd = {k: v.float() for k, v in torch.load(path, map_location="cpu")["weight"].items()}
                cur = net.state_dict()
                with torch.no_grad():          # in place: parameters are views into the flat optimizer arenas
                    missing = [k for k in cur if k not in sd]
                    if strict and missing:
                        raise RuntimeError(f"pretrained checkpoint {path} lacks {missing[:4]}...")
                    for k, v in cur.items():
                        if k in sd:
                            v.copy_(sd[k])
                logger.info("loaded pretrained %s", path)
            else:
                logger.warning("no pretrained weights at %r: training this network from random initialisation", path)

    def _run(self, rank, world, local_rank):
        hps, t = self.hps, self.hps["train"]
        device = torch.device("cuda", local_rank)
        torch.cuda.set_device(device)
        if world > 1 and not dist.is_initialized():
            dist.init_process_group("nccl", rank=rank, world_size=world, device_id=device)
        net_g, net_d = self._build(device)
        step = s2_step.S2Step(net_g, net_d, t, hps["data"], world_size=world)
        ops.manual_seed(t["seed"] + rank)
        dataset = self.dataset or s2data.TextAudioSpeakerLoader(hps["data"]["exp_dir"], hps["data"]["sampling_rate"],
                                                                 hps["data"]["hop_length"])
        sampler = s2data.DistributedBucketSampler(dataset.lengths, t["batch_size"], BUCKET_BOUNDARIES, world, rank, True)
        loader = torch.utils.data.DataLoader(dataset, num_workers=2, pin_memory=True, batch_sampler=sampler,
                                             collate_fn=s2data.TextAudioSpeakerCollate(hps["data"]["hop_length"]))
        epoch_str = 1
        logs = t["train_logs_dir"]
        try:                                                          # resume, sovits.py:327-343
            path_d, path_g = ckpt.latest_checkpoint_path(logs, "D_*.pth"), ckpt.latest_checkpoint_path(logs, "G_*.pth")
        except IndexError:                                            # no resumable checkpoint: the only case that falls
            path_d = path_g = None                                    # through to the pretrained weights (sovits.py:344-366)
        if path_g is not None:
            _, _, _, epoch_str = ckpt.load_checkpoint(path_d, net_d, step.opt_d)
            _, _, _, epoch_str = ckpt.load_checkpoint(path_g, net_g, step.opt_g)
            self.global_step = (epoch_str - 1) * len(loader)
            step.lr = step.opt_g.lr_host                              # the reference continues from the lr stored in the optimizer
            logger.info("resumed from %s (epoch %d)", path_g, epoch_str)
        else:
            epoch_str, self.global_step = 1, 0
            self._load_pretrained(net_g, net_d)
        step.set_lr(step.lr * t["lr_decay"] ** epoch_str)             # ExponentialLR fast-forward (sovits.py:368-376)
        connector = MultiProcessOutputConnector()
        writer = None
        if rank == 0:                                                 # sovits.py:217
            from torch.utils.tensorboard.writer import SummaryWriter
            writer = SummaryWriter(log_dir=tensorboard_log_dir(hps["name"]))
        hop = hps["data"]["hop_length"]
        for epoch in range(epoch_str, t["epochs"] + 1):
            sampler.set_epoch(epoch)
            for host in loader:
                Tq, Xq = step.agree_shape(host["ssl"].shape[2], host["text"].shape[1])
                host = s2data_pad(host, Tq, Xq, hop)
                batch = s2_step.to_device_batch(host, device, step.bank, hop)
                out = step.train_step(batch)
                gs = self.global_step
                if gs % 10 == 0:                                      # sovits.py:527-536
                    lg, ld = float(out["loss_gen_all"]), float(out["loss_disc"])
                    if rank == 0:
                        connector.write_loss(gs, loss=lg, other={"loss/g/total": lg, "loss/d/total": ld, "learning_rate": step.lr})
                if writer is not None and gs % 5 == 0:                # sovits.py:538-568 (helper.summarize)
                    scalars = {"loss/g/total": float(out["loss_gen_all"]), "loss/d/total": float(out["loss_disc"]),
                               "learning_rate": step.lr, "grad_norm_d": float(out["grad_norm_d"]) ** 0.5,
                               "grad_norm_g": float(out["grad_norm_g"]) ** 0.5, "loss/g/fm": float(out["loss_fm"]),
                               "loss/g/mel": float(out["loss_mel"]), "loss/g/kl_ssl": 0.0, "loss/g/kl": float(out["loss_kl"])}
                    for k, v in scalars.items():
                        writer.add_scalar(k, v, gs)
                    writer.flush()
                self.global_step += 1
            if rank == 0 and epoch % t["save_every_epoch"] == 0:
                self._save(epoch, net_g, net_d, step)
            step.decay_lr()
        if writer is not None:
            writer.flush()
            writer.close()
        if world > 1:
            dist.barrier()

    def _save(self, epoch, net_g, net_d, step):
        t = self.hps["train"]
        tag = "latest" if t["if_save_latest"] else str(self.global_step)
        ckpt.save_checkpoint(net_g, step.opt_g, t["learning_rate"], epoch, os.path.join(t["train_logs_dir"], f"G_{tag}.pth"))
        ckpt.save_checkpoint(net_d, step.opt_d, t["learning_rate"], epoch, os.path.join(t["train_logs_dir"], f"D_{tag}.pth"))
        if t["if_save_every_weights"]:
            ckpt.export_weights(net_g.state_dict(), self.hps, f"{self.hps['name']}_e{epoch}_s{self.global_step}", epoch,
                                self.global_step, t["save_weight_dir"])


def _spawn_entry(local_rank, world, params, gpu_ids, dataset=None):
    os.environ.update(RANK=str(local_rank), WORLD_SIZE=str(world), LOCAL_RANK=str(gpu_ids[local_rank]))
    SovitsTrain(params, dataset=dataset).train()
