#!/usr/bin/env python
"""Pretraining driver with the reference's command line (THUDM/GCC train.py:40-130, pretraining
flags only) on the H100-native hot path.

    python train.py --moco --nce-k 16384 --dataset synthetic-chunglu --graph-nodes 1000000 \
        --graph-edges 20000000 --batch-size 256 --epochs 1 --num-samples 2000 --num-workers 12
    torchrun --nproc-per-node 8 train.py --moco --nce-k 16384 ...          (one process per GPU)

What it keeps from the reference: flag names and defaults, run naming (train.py:133-166), the
triangular LR schedule with 10% warm-up (train.py:411-416, gcc/utils/misc.py:5-10), BatchNorm of the
momentum encoder in train mode (train.py:357-365), the checkpoint dict
{"opt","model","contrast","optimizer","epoch","model_ema"} with the reference's state_dict keys
(train.py:748-786; "optimizer" is the state_dict of the torch.optim.SGD / Adam / Adagrad that --optimizer
names, over model.parameters(), built from the flat optimiser buffers), print/TensorBoard scalars (train.py:438-472), and the reference's step indexing:
epochs are 1-based and global_step = epoch * n_batch + idx (train.py:411,733), so the LR schedule starts
one epoch into its warm-up exactly like the reference's.  What changes: the data loader and the whole
step run on the GPU through gcc_b200.engine.PretrainEngine (no DataLoader workers, no .item() per step:
loss / prob / grad-norm are accumulated on the device EVERY step and read every --print-freq steps, so
the meters average over all steps like the reference's).

Fine-tuning (--finetune, train.py:175-337,516-545,631-660,788-792 of the reference): main_finetune drives
gcc_b200.finetune.FinetuneEngine -- every step on the device with no host sync: the batch, the encoder, the head's
cross-entropy and micro-F1, clip_grad_value_(1), the --optimizer for the encoder and Adam for the output layer --
over the labeled datasets of gcc_b200/datasets/labeled.py, split by the reference's StratifiedKFold(10, shuffle,
seed)[fold_idx].  train_finetune / test_finetune keep the reference's signatures and torch-ops arithmetic
(GraphEncoder forward/backward through the same device kernels as an autograd Function, torch's Linear head,
CrossEntropyLoss, torch.optim): they compute the same steps on the same batches and are what the engine is tested
against.

    python train.py --finetune --dataset usa_airport --resume saved/.../current.pth --epochs 30 --fold-idx 0
"""
import argparse
import os
import time

import numpy as np
import torch

from gcc_b200.contrastive.memory_moco import MemoryMoCo
from gcc_b200.datasets import downstream, synthetic
from gcc_b200.datasets.graph_dataset import (GraphClassificationDataset, LoadBalanceGraphDataset,
                                             NodeClassificationDataset)
from gcc_b200.engine import PretrainEngine
from gcc_b200.finetune import FinetuneEngine
from gcc_b200.models import GraphEncoder
from gcc_b200.utils.misc import AverageMeter, warmup_linear


def parse_option(argv=None):
    # fmt: off
    parser = argparse.ArgumentParser("argument for training")
    parser.add_argument("--print-freq", type=int, default=10, help="print frequency")
    parser.add_argument("--tb-freq", type=int, default=250, help="tb frequency")
    parser.add_argument("--save-freq", type=int, default=1, help="save frequency")
    parser.add_argument("--batch-size", type=int, default=32, help="batch_size")
    parser.add_argument("--num-workers", type=int, default=12, help="num of workers to use (sizes an epoch: total = num_samples * num_workers)")
    parser.add_argument("--num-copies", type=int, default=6, help="num of dataset copies that fit in memory")
    parser.add_argument("--num-samples", type=int, default=2000, help="num of samples per batch per worker")
    parser.add_argument("--epochs", type=int, default=100, help="number of training epochs")
    # optimization
    parser.add_argument("--optimizer", type=str, default="adam", choices=["sgd", "adam", "adagrad"], help="optimizer")
    parser.add_argument("--learning_rate", type=float, default=0.005, help="learning rate")
    parser.add_argument("--lr_decay_epochs", type=str, default="120,160,200", help="where to decay lr, can be a list")
    parser.add_argument("--lr_decay_rate", type=float, default=0.0, help="decay rate for learning rate (Adagrad's lr_decay)")
    parser.add_argument("--beta1", type=float, default=0.9, help="beta1 for adam")
    parser.add_argument("--beta2", type=float, default=0.999, help="beta2 for Adam")
    parser.add_argument("--weight-decay", type=float, default=1e-5, help="weight decay")
    parser.add_argument("--momentum", type=float, default=0.9, help="momentum (SGD)")
    parser.add_argument("--clip-norm", type=float, default=1.0, help="clip norm")
    parser.add_argument("--resume", default="", type=str, metavar="PATH", help="path to latest checkpoint")
    parser.add_argument("--exp", type=str, default="")
    # dataset definition
    parser.add_argument("--dataset", type=str, default="synthetic-chunglu",
                        help="synthetic-chunglu | synthetic-er | dgl (./data/small.bin) | a downstream node or graph "
                             "dataset (%s; files under ./data) | path to .npz(indptr, indices[, graph_sizes]) or DGL "
                             ".bin" % ", ".join(downstream.NODE_DSETS + downstream.GRAPH_DSETS))
    parser.add_argument("--graph-nodes", type=int, default=1000000)
    parser.add_argument("--graph-edges", type=int, default=20000000)
    # model definition
    parser.add_argument("--model", type=str, default="gin", choices=["gin", "gat"])
    parser.add_argument("--num-layer", type=int, default=5, help="gnn layers")
    parser.add_argument("--readout", type=str, default="avg", choices=["avg", "set2set"])
    parser.add_argument("--set2set-lstm-layer", type=int, default=3, help="lstm layers for s2s")
    parser.add_argument("--set2set-iter", type=int, default=6, help="s2s iteration")
    parser.add_argument("--norm", action="store_true", default=True, help="apply 2-norm on output feats")
    # loss function
    parser.add_argument("--nce-k", type=int, default=32)
    parser.add_argument("--nce-t", type=float, default=0.07)
    # random walk
    parser.add_argument("--rw-hops", type=int, default=256)
    parser.add_argument("--subgraph-size", type=int, default=128)
    parser.add_argument("--restart-prob", type=float, default=0.8)
    parser.add_argument("--hidden-size", type=int, default=64)
    parser.add_argument("--positional-embedding-size", type=int, default=32)
    parser.add_argument("--max-node-freq", type=int, default=16)
    parser.add_argument("--max-edge-freq", type=int, default=16)
    parser.add_argument("--max-degree", type=int, default=512)
    parser.add_argument("--freq-embedding-size", type=int, default=16)
    parser.add_argument("--degree-embedding-size", type=int, default=16)
    # specify folder
    parser.add_argument("--model-path", type=str, default="saved", help="path to save model")
    parser.add_argument("--tb-path", type=str, default="tensorboard", help="path to tensorboard")
    # memory setting
    parser.add_argument("--moco", action="store_true", help="using MoCo (otherwise Instance Discrimination)")
    parser.add_argument("--alpha", type=float, default=0.999, help="exponential moving average weight")
    parser.add_argument("--gpu", default=None, type=int, nargs="+", help="GPU id to use.")
    parser.add_argument("--seed", type=int, default=0, help="random seed.")
    parser.add_argument("--max-steps", type=int, default=0, help="stop after this many steps (0 = full run)")
    # finetune setting / cross validation (train.py:109-120)
    parser.add_argument("--finetune", action="store_true")
    parser.add_argument("--fold-idx", type=int, default=0, help="fold of the 10-fold stratified split")
    parser.add_argument("--cv", action="store_true", help="run all 10 folds and print mean / std of the micro-F1")
    # fmt: on
    opt = parser.parse_args(argv)
    opt.lr_decay_epochs = [int(it) for it in opt.lr_decay_epochs.split(",")]      # train.py:125-128
    return opt


def option_update(opt):
    """Run naming of the reference (train.py:133-166)."""
    ft = bool(getattr(opt, "finetune", False))
    prefix = ("FT_{}" if ft else "Pretrain_{}").format(opt.exp) if opt.exp else ("FT" if ft else "Pretrain")
    opt.model_name = "{}_{}_{}_{}_layer_{}_lr_{}_decay_{}_bsz_{}_hid_{}_samples_{}_nce_t_{}_nce_k_{}_rw_hops_{}_restart_prob_{}_aug_1st_ft_{}_deg_{}_pos_{}_momentum_{}".format(
        prefix, "moco" if opt.moco else "e2e", os.path.basename(str(opt.dataset)), opt.model, opt.num_layer,
        opt.learning_rate, opt.weight_decay, opt.batch_size, opt.hidden_size, opt.num_samples, opt.nce_t,
        opt.nce_k, opt.rw_hops, opt.restart_prob, ft, opt.degree_embedding_size, opt.positional_embedding_size,
        opt.alpha)
    opt.model_folder = os.path.join(opt.model_path, opt.model_name)
    os.makedirs(opt.model_folder, exist_ok=True)
    opt.tb_folder = os.path.join(opt.tb_path, opt.model_name)
    os.makedirs(opt.tb_folder, exist_ok=True)
    return opt


def build_graph(args, device):
    if args.dataset == "synthetic-chunglu":
        return synthetic.chung_lu_device(args.graph_nodes, args.graph_edges, 0.5, seed=0, device=device)
    if args.dataset == "synthetic-er":
        return synthetic.erdos_renyi(args.graph_nodes, args.graph_edges, seed=0)
    if args.dataset == "dgl":
        return "./data/small.bin"    # the reference's default pretraining corpus (train.py:547-556)
    return args.dataset          # path to .npz or .bin


def build_dataset(args, device):
    """The reference's three branches (train.py:547-573): a downstream node dataset (every node of its multigraph
    in order), a TU graph dataset (every whole graph in order), else the sampled ego-nets of
    LoadBalanceGraphDataset over the corpus build_graph names."""
    kw = dict(rw_hops=args.rw_hops, restart_prob=args.restart_prob,
              positional_embedding_size=args.positional_embedding_size, batch_size=args.batch_size, seed=args.seed,
              device=device)
    if args.dataset in downstream.NODE_DSETS:
        return NodeClassificationDataset(downstream.node_dataset_graph(args.dataset),
                                         subgraph_size=args.subgraph_size, **kw)
    if args.dataset in downstream.GRAPH_DSETS:
        return GraphClassificationDataset(args.dataset, subgraph_size=args.subgraph_size, **kw)
    return LoadBalanceGraphDataset(num_workers=args.num_workers, num_samples=args.num_samples,
                                   dgl_graphs_file=build_graph(args, device), num_copies=args.num_copies, **kw)


def train_moco(epoch, engine, sw, opt, is_main):
    """One epoch (train.py:350-478): n_batch = dataset.total // batch_size steps.  A node or graph dataset also
    trains its last total mod batch_size items as a short batch (the reference's DataLoader keeps it); the LR
    schedule keeps n_batch, so that batch runs at idx = n_batch."""
    n_batch = engine.ds.total // (opt.batch_size * engine.world)
    if n_batch == 0:
        raise ValueError("dataset.total = %d is smaller than one global batch (%d x %d): nothing to train on"
                         % (engine.ds.total, opt.batch_size, engine.world))
    n_steps = engine.ds.steps_per_epoch() if getattr(engine.ds, "epoch_ordered", False) else n_batch
    loss_meter, prob_meter, gs_meter, gnorm_meter = (AverageMeter() for _ in range(4))
    epoch_loss, batch_time = AverageMeter(), AverageMeter()
    end = time.time()
    max_nodes = max_edges = 0
    for idx in range(n_steps):
        global_step = epoch * n_batch + idx
        lr = opt.learning_rate * warmup_linear(global_step / (opt.epochs * n_batch), 0.1)   # train.py:411-416
        engine.step(lr=lr)
        if (idx + 1) % opt.print_freq == 0 or idx + 1 == n_steps:
            s = engine.read_stats()                      # the only host sync of the window
            bsz = s["batch_size"]                        # of the last step: opt.batch_size but for a short batch
            w = max(s["window_steps"], 1)                # device-side sums over every step since the last read
            pairs = s["window_pairs"]                    # the meters weight each step by its pairs, as the reference
            loss_meter.update(s["window_loss"], pairs)
            epoch_loss.update(s["window_loss"], pairs)
            prob_meter.update(s["window_prob"], pairs)
            gs_meter.update((s["nodes_q"] + s["nodes_k"]) / 2.0 / bsz, 2 * bsz)
            gnorm_meter.update(s["window_grad_norm"], w)
            max_nodes, max_edges = max(max_nodes, s["nodes_q"]), max(max_edges, s["edges_q"])
            batch_time.update((time.time() - end) / opt.print_freq)
            end = time.time()
            if is_main:
                print("Train: [{0}][{1}/{2}]\tBT {bt.val:.4f} ({bt.avg:.4f})\tloss {loss.val:.3f} ({loss.avg:.3f})\t"
                      "prob {prob.val:.3f} ({prob.avg:.3f})\tGS {gs.val:.3f} ({gs.avg:.3f})\tlr {lr:.6f}".format(
                          epoch, idx + 1, n_steps, bt=batch_time, loss=loss_meter, prob=prob_meter, gs=gs_meter, lr=lr))
        if sw is not None and (idx + 1) % opt.tb_freq == 0:
            sw.add_scalar("moco_loss", loss_meter.avg, global_step)
            sw.add_scalar("moco_prob", prob_meter.avg, global_step)
            sw.add_scalar("graph_size", gs_meter.avg, global_step)
            sw.add_scalar("graph_size/max", max_nodes, global_step)
            sw.add_scalar("graph_size/max_edges", max_edges, global_step)
            sw.add_scalar("gnorm", gnorm_meter.avg, global_step)
            sw.add_scalar("learning_rate", lr, global_step)
            for m in (loss_meter, prob_meter, gs_meter, gnorm_meter):
                m.reset()
            max_nodes = max_edges = 0
        if opt.max_steps and engine.global_step >= opt.max_steps:
            break
    return epoch_loss.avg


class LabeledLoader:
    """What DataLoader(Subset(dataset, idx), batch_size, collate_fn=labeled_batcher(), shuffle=...) is to the
    reference (train.py:543-545,576-592): an iterable of (graph_q, y) with a length in batches."""

    def __init__(self, dataset, indices, batch_size, shuffle, seed=0):
        self.dataset, self.indices, self.batch_size, self.shuffle = dataset, np.asarray(indices), batch_size, shuffle
        self.rng = np.random.RandomState(seed)

    def __len__(self):
        return self.dataset.num_batches(len(self.indices), self.batch_size)

    def __iter__(self):
        return self.dataset.batches(self.indices, self.batch_size, self.shuffle, self.rng)


def train_finetune(epoch, train_loader, model, output_layer, criterion, optimizer, output_layer_optimizer, sw, opt):
    """One finetune epoch (train.py:175-297): same order of operations as the reference."""
    from sklearn.metrics import f1_score
    n_batch = len(train_loader)
    model.train()
    output_layer.train()
    batch_time, loss_meter, f1_meter = AverageMeter(), AverageMeter(), AverageMeter()
    epoch_loss_meter, epoch_f1_meter, graph_size = AverageMeter(), AverageMeter(), AverageMeter()
    max_num_nodes = max_num_edges = 0
    end = time.time()
    for idx, (graph_q, y) in enumerate(train_loader):
        bsz = graph_q.batch_size
        feat_q = model(graph_q)
        assert feat_q.shape == (bsz, opt.hidden_size)
        out = output_layer(feat_q)
        loss = criterion(out, y)
        optimizer.zero_grad()
        output_layer_optimizer.zero_grad()
        loss.backward()
        torch.nn.utils.clip_grad_value_(model.parameters(), 1)
        torch.nn.utils.clip_grad_value_(output_layer.parameters(), 1)
        global_step = epoch * n_batch + idx
        lr_this_step = opt.learning_rate * warmup_linear(global_step / (opt.epochs * n_batch), 0.1)
        for group in list(optimizer.param_groups) + list(output_layer_optimizer.param_groups):
            group["lr"] = lr_this_step
        optimizer.step()
        output_layer_optimizer.step()
        preds = out.argmax(dim=1)
        f1 = f1_score(y.cpu().numpy(), preds.cpu().numpy(), average="micro")
        f1_meter.update(f1, bsz)
        epoch_f1_meter.update(f1, bsz)
        loss_meter.update(loss.item(), bsz)
        epoch_loss_meter.update(loss.item(), bsz)
        graph_size.update(graph_q.number_of_nodes() / bsz, bsz)
        max_num_nodes = max(max_num_nodes, graph_q.number_of_nodes())
        max_num_edges = max(max_num_edges, graph_q.number_of_edges())
        batch_time.update(time.time() - end)
        end = time.time()
        if (idx + 1) % opt.print_freq == 0:
            print("Train: [{0}][{1}/{2}]\tBT {bt.val:.3f} ({bt.avg:.3f})\tloss {loss.val:.3f} ({loss.avg:.3f})\t"
                  "f1 {f1.val:.3f} ({f1.avg:.3f})\tGS {gs.val:.3f} ({gs.avg:.3f})".format(
                      epoch, idx + 1, n_batch, bt=batch_time, loss=loss_meter, f1=f1_meter, gs=graph_size))
        if sw is not None and (idx + 1) % opt.tb_freq == 0:
            sw.add_scalar("ft_loss", loss_meter.avg, global_step)
            sw.add_scalar("ft_f1", f1_meter.avg, global_step)
            sw.add_scalar("graph_size", graph_size.avg, global_step)
            sw.add_scalar("lr", lr_this_step, global_step)
            sw.add_scalar("graph_size/max", max_num_nodes, global_step)
            sw.add_scalar("graph_size/max_edges", max_num_edges, global_step)
            loss_meter.reset()
            f1_meter.reset()
            graph_size.reset()
            max_num_nodes = max_num_edges = 0
    return epoch_loss_meter.avg, epoch_f1_meter.avg


def test_finetune(epoch, valid_loader, model, output_layer, criterion, sw, opt):
    """Validation pass (train.py:300-337): eval-mode encoder (running BatchNorm statistics, no dropout)."""
    from sklearn.metrics import f1_score
    n_batch = len(valid_loader)
    model.eval()
    output_layer.eval()
    epoch_loss_meter, epoch_f1_meter = AverageMeter(), AverageMeter()
    for idx, (graph_q, y) in enumerate(valid_loader):
        bsz = graph_q.batch_size
        with torch.no_grad():
            feat_q = model(graph_q)
            assert feat_q.shape == (bsz, opt.hidden_size)
            out = output_layer(feat_q)
        loss = criterion(out, y)
        preds = out.argmax(dim=1)
        f1 = f1_score(y.cpu().numpy(), preds.cpu().numpy(), average="micro")
        epoch_loss_meter.update(loss.item(), bsz)
        epoch_f1_meter.update(f1, bsz)
    global_step = (epoch + 1) * n_batch
    if sw is not None:
        sw.add_scalar("ft_loss/valid", epoch_loss_meter.avg, global_step)
        sw.add_scalar("ft_f1/valid", epoch_f1_meter.avg, global_step)
    print(f"Epoch {epoch}, loss {epoch_loss_meter.avg:.3f}, f1 {epoch_f1_meter.avg:.3f}")
    return epoch_loss_meter.avg, epoch_f1_meter.avg


def make_optimizer(args, params):
    """The encoder optimiser --optimizer names (train.py:659-681).  --lr_decay_epochs is parsed but, as in the
    reference, unused: the per-step warm-up LR overwrites what adjust_learning_rate would set."""
    if args.optimizer == "sgd":
        return torch.optim.SGD(params, lr=args.learning_rate, momentum=args.momentum, weight_decay=args.weight_decay)
    if args.optimizer == "adam":
        return torch.optim.Adam(params, lr=args.learning_rate, betas=(args.beta1, args.beta2),
                                weight_decay=args.weight_decay)
    if args.optimizer == "adagrad":
        return torch.optim.Adagrad(params, lr=args.learning_rate, lr_decay=args.lr_decay_rate,
                                   weight_decay=args.weight_decay)
    raise NotImplementedError(args.optimizer)


def _make_encoder(args):
    return GraphEncoder(positional_embedding_size=args.positional_embedding_size, max_node_freq=args.max_node_freq,
                        max_edge_freq=args.max_edge_freq, max_degree=args.max_degree,
                        freq_embedding_size=args.freq_embedding_size,
                        degree_embedding_size=args.degree_embedding_size, output_dim=args.hidden_size,
                        node_hidden_dim=args.hidden_size, edge_hidden_dim=args.hidden_size,
                        num_layers=args.num_layer, num_step_set2set=args.set2set_iter,
                        num_layer_set2set=args.set2set_lstm_layer, norm=args.norm, gnn_model=args.model,
                        degree_input=True)


def main_finetune(args, dataset=None):
    """The --finetune branch of the reference's main (train.py:483-545,600-660,716-792): hyper-parameters come
    from the pretraining checkpoint, 10-fold stratified split, BatchNorm running statistics reset, the
    --optimizer for the encoder and Adam for the output layer, validation after the last epoch.  Returns the validation micro-F1."""
    from sklearn.model_selection import StratifiedKFold

    from gcc_b200.datasets.labeled import (GRAPH_CLASSIFICATION_DSETS, GraphClassificationDatasetLabeled,
                                           NodeClassificationDatasetLabeled)
    dev = torch.device("cuda", args.gpu[0] if isinstance(args.gpu, (list, tuple)) and args.gpu else (args.gpu or 0))
    torch.cuda.set_device(dev)
    np.random.seed(args.seed)
    torch.manual_seed(args.seed)
    torch.cuda.manual_seed(args.seed)
    checkpoint = None
    if args.resume:
        if os.path.isfile(args.resume):
            print("=> loading checkpoint '{}'".format(args.resume))
            checkpoint = torch.load(args.resume, map_location="cpu", weights_only=False)
            pre = checkpoint["opt"]                        # train.py:491-504: the pretraining run's options win
            for k in ("fold_idx", "gpu", "finetune", "resume", "cv", "dataset", "epochs", "num_workers", "batch_size"):
                setattr(pre, k, getattr(args, k))
            for k, v in vars(args).items():                # options this driver has and an older checkpoint lacks
                if not hasattr(pre, k):
                    setattr(pre, k, v)
            args = pre
        else:
            print("=> no checkpoint found at '{}'".format(args.resume))
    args = option_update(args)
    if dataset is None:
        kw = dict(dataset=args.dataset, rw_hops=args.rw_hops, subgraph_size=args.subgraph_size,
                  restart_prob=args.restart_prob, positional_embedding_size=args.positional_embedding_size,
                  device=dev, seed=args.seed, batch_size=args.batch_size)
        dataset = (GraphClassificationDatasetLabeled(**kw) if args.dataset in GRAPH_CLASSIFICATION_DSETS
                   else NodeClassificationDatasetLabeled(**kw))
    labels = dataset.labels.tolist()
    skf = StratifiedKFold(n_splits=10, shuffle=True, random_state=args.seed)
    idx_list = list(skf.split(np.zeros(len(labels)), labels))
    assert 0 <= args.fold_idx < 10, "fold_idx must be from 0 to 9."
    train_idx, test_idx = idx_list[args.fold_idx]
    model = _make_encoder(args)
    if checkpoint is not None:
        model.load_state_dict(checkpoint["model"])
    model = model.to(dev)
    output_layer = torch.nn.Linear(in_features=args.hidden_size, out_features=dataset.num_classes).to(dev)

    def clear_bn(m):                                       # train.py:648-653
        if m.__class__.__name__.find("BatchNorm") != -1:
            m.reset_running_stats()

    model.apply(clear_bn)
    # the --optimizer for the encoder, Adam for the output layer, both after clip_grad_value_(1), every step on the
    # device (gcc_b200/finetune.py); train_finetune / test_finetune are the same steps with torch ops
    engine = FinetuneEngine(dataset, model, output_layer, optimizer=args.optimizer, lr=args.learning_rate,
                            betas=(args.beta1, args.beta2), weight_decay=args.weight_decay, momentum=args.momentum,
                            lr_decay=args.lr_decay_rate, batch_size=args.batch_size)
    rng = np.random.RandomState(args.seed)                 # LabeledLoader's shuffle: one permutation per epoch
    sw = None
    try:
        from torch.utils.tensorboard import SummaryWriter
        sw = SummaryWriter(args.tb_folder)
    except Exception:
        sw = None
    epoch = 0
    for epoch in range(1, args.epochs + 1):
        t0 = time.time()
        loss, _ = engine.train_epoch(epoch, rng.permutation(np.asarray(train_idx, dtype=np.int64)), args.epochs,
                                     sw=sw, print_freq=args.print_freq, tb_freq=args.tb_freq)
        print("epoch {}, loss {:.4f}, total time {:.2f}".format(epoch, loss, time.time() - t0))
        state = {"opt": args, "model": model.state_dict(), "optimizer": engine.optimizer_state_dict(),
                 "epoch": epoch}
        torch.save(state, os.path.join(args.model_folder, "current.pth"))
        if epoch % args.save_freq == 0:
            torch.save(state, os.path.join(args.model_folder, "ckpt_epoch_{epoch}.pth".format(epoch=epoch)))
    _, valid_f1 = engine.evaluate(epoch, test_idx, sw)
    return valid_f1


def main(args):
    if getattr(args, "finetune", False):
        return main_finetune(args)
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", str(args.gpu[0] if args.gpu else 0)))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        torch.distributed.init_process_group("nccl", device_id=dev)
    np.random.seed(args.seed)
    torch.manual_seed(args.seed)
    torch.cuda.manual_seed(args.seed)
    args = option_update(args)
    train_dataset = build_dataset(args, dev)
    model, model_ema = [
        GraphEncoder(positional_embedding_size=args.positional_embedding_size, max_node_freq=args.max_node_freq,
                     max_edge_freq=args.max_edge_freq, max_degree=args.max_degree,
                     freq_embedding_size=args.freq_embedding_size,
                     degree_embedding_size=args.degree_embedding_size, output_dim=args.hidden_size,
                     node_hidden_dim=args.hidden_size, edge_hidden_dim=args.hidden_size,
                     num_layers=args.num_layer, num_step_set2set=args.set2set_iter,
                     num_layer_set2set=args.set2set_lstm_layer, norm=args.norm, gnn_model=args.model,
                     degree_input=True) for _ in range(2)]
    if args.moco:
        model_ema.load_state_dict(model.state_dict())          # moment_update(model, model_ema, 0), train.py:623-624
    contrast = MemoryMoCo(args.hidden_size, None, args.nce_k, args.nce_t, use_softmax=True)
    start_epoch = 1
    if args.resume:
        ckpt = torch.load(args.resume, map_location="cpu", weights_only=False)
        model.load_state_dict(ckpt["model"])
        contrast.load_state_dict(ckpt["contrast"])
        if args.moco and "model_ema" in ckpt:
            model_ema.load_state_dict(ckpt["model_ema"])
        # like the reference (train.py:689-691) the optimiser state and start epoch are NOT restored
    model, model_ema, contrast = model.to(dev), model_ema.to(dev), contrast.to(dev)
    engine = PretrainEngine(train_dataset, model, model_ema, contrast, moco=args.moco,
                            learning_rate=args.learning_rate, betas=(args.beta1, args.beta2),
                            weight_decay=args.weight_decay, clip_norm=args.clip_norm, alpha=args.alpha,
                            nce_t=args.nce_t, rank=rank, world_size=world, optimizer=args.optimizer,
                            momentum=args.momentum, lr_decay=args.lr_decay_rate)
    sw = None
    if rank == 0:
        try:
            from torch.utils.tensorboard import SummaryWriter
            sw = SummaryWriter(args.tb_folder)
        except Exception:
            sw = None
    for epoch in range(start_epoch, args.epochs + 1):
        t0 = time.time()
        loss = train_moco(epoch, engine, sw, args, rank == 0)        # 1-based, as the reference (train.py:733)
        if rank == 0:
            print("epoch {}, loss {:.4f}, total time {:.2f}".format(epoch, loss, time.time() - t0))
            if epoch % args.save_freq == 0:
                state = {"opt": args, "model": model.state_dict(), "contrast": contrast.state_dict(),
                         "optimizer": engine.optimizer_state_dict(),
                         "epoch": epoch}
                if args.moco:
                    state["model_ema"] = model_ema.state_dict()
                torch.save(state, os.path.join(args.model_folder, "ckpt_epoch_{epoch}.pth".format(epoch=epoch)))
                torch.save(state, os.path.join(args.model_folder, "current.pth"))
        if args.max_steps and engine.global_step >= args.max_steps:
            break
    if world > 1:
        torch.distributed.destroy_process_group()


if __name__ == "__main__":
    _args = parse_option()
    if _args.cv and _args.finetune:                         # train.py:801-816
        import copy
        f1 = []
        for fold_idx in range(10):
            a = copy.deepcopy(_args)
            a.fold_idx = fold_idx
            f1.append(main(a))
        print(f1)
        print(f"Mean = {np.mean(f1)}; Std = {np.std(f1)}")
    else:
        main(_args)
