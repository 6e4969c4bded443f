"""N-rank equivalence checks (run under torchrun, one rank per GPU):
 (1) all-reduce path: the reduced gradient on every rank equals the mean of the single-rank gradients computed with the same
     weights on each rank's clip, bit-identical across ranks;
 (2) sharded path (ShardedAdamW: reduce-scatter + AdamW on 1/N + bf16 all-gather): after one step every rank holds the same
     bf16 operand weights, equal to those of the all-reduce + replicated FusedAdamW step, and gather_masters() restores the
     fp32 masters everywhere;
 (3) the same step as ONE kernel over NVLink peer memory (P2PShardedAdamW), eager and replayed from a CUDA graph;
 (4) checkpoint and resume of ShardedAdamW: train at world N, state_dict() (collective), continue; a fresh optimizer that loads
     the dict at world N continues bit for bit, and one at world N/2 (a subgroup) ends on masters within the tolerance of (2);
 (5) the sharded 8-bit forms (ShardedAdamW8bit, P2PShardedAdamW8bit) against FusedAdamW8bit.step(1/N) over the rank-order sum of
     the ranks' gradients, three steps: the P2P form bit for bit, the NCCL form (whose reduce-scatter sums in its own order)
     within the tolerance of (2); every rank's operands identical; state_dict() (collective) equal to FusedAdamW8bit's."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.distributed as dist

from svd_xtend_b200.train import (FusedAdamW, FusedAdamW8bit, GradReducer, P2PShardedAdamW, P2PShardedAdamW8bit, ParamArena,
                                  ShardedAdamW, ShardedAdamW8bit)
from svd_xtend_b200.unet import UNetSpatioTemporalConditionModel
from svd_xtend_b200.workload import edm_loss, synthetic_batch

TINY = dict(sample_size=None, in_channels=8, out_channels=4,
            down_block_types=("CrossAttnDownBlockSpatioTemporal", "DownBlockSpatioTemporal"),
            up_block_types=("UpBlockSpatioTemporal", "CrossAttnUpBlockSpatioTemporal"),
            block_out_channels=(64, 128), addition_time_embed_dim=32, projection_class_embeddings_input_dim=96, layers_per_block=1,
            cross_attention_dim=64, transformer_layers_per_block=1, num_attention_heads=(1, 2), num_frames=4)

rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(local)
dev = torch.device("cuda", local)
dist.init_process_group("nccl", device_id=dev)


def build(pad_world=None, block=64):
    torch.manual_seed(0)
    unet = UNetSpatioTemporalConditionModel(**TINY).to(dev)
    unet.requires_grad_(False)
    for n, p in unet.named_parameters():
        if "temporal_transformer_block" in n:
            p.requires_grad_(True)
    unet.train()
    arena = ParamArena(unet, pad_to=(pad_world or world) * (256 if block == 256 else 64), block=block)
    unet.attach_arena(arena)
    return unet, arena


def backward(unet, arena, seed):
    b = synthetic_batch(1, 4, 16, 16, seed=seed, device=dev, cross_dim=TINY["cross_attention_dim"])
    arena.zero_grad()
    pred = unet(b["sample"], b["timestep"], b["encoder_hidden_states"], b["added_time_ids"]).sample
    edm_loss(pred.float(), b["noisy"], b["latents"], b["sigmas"]).backward()


# ---- (1) all-reduce path
unet, arena = build()
red = GradReducer(arena, bucket_mb=0.5)
unet.grad_hook = lambda ps: red.on_grads_ready(ps) if ps is not None else None
backward(unet, arena, 100 + rank)
red.finish()
torch.cuda.synchronize()
g_red = arena.grad.clone()
unet.grad_hook = None
singles = []
for r in range(world):
    backward(unet, arena, 100 + r)
    torch.cuda.synchronize()
    singles.append(arena.grad.clone())
ref = sum(singles) / world
rel = ((g_red - ref).norm() / ref.norm()).item()
others = [torch.empty_like(g_red) for _ in range(world)]
dist.all_gather(others, g_red)
same = all(torch.equal(o, g_red) for o in others)
print(f"[ddp_check] rank {rank}: all-reduce path: reduced-vs-mean rel-l2 {rel:.3e}, identical across ranks: {same}, buckets {len(red.buckets)}", flush=True)
assert rel < 2e-2 and same

# ---- (2) sharded path vs all-reduce + replicated AdamW, same gradients
w0 = arena.data.clone()
arena.grad.copy_(singles[rank])
opt_ref = FusedAdamW(arena, lr=1e-3, weight_decay=1e-2)
dist.all_reduce(arena.grad)
arena.grad.mul_(1.0 / world)
opt_ref.step()
torch.cuda.synchronize()
shadow_ref, data_ref = arena.shadow.clone(), arena.data.clone()

arena.data.copy_(w0)
arena.refresh_shadow()
arena.grad.copy_(singles[rank])
opt = ShardedAdamW(arena, lr=1e-3, weight_decay=1e-2)
opt.step()
torch.cuda.synchronize()
upd_ref = (shadow_ref.float() - w0)
upd = (arena.shadow.float() - w0)
e_shadow = ((upd - upd_ref).norm() / upd_ref.norm()).item()
others = [torch.empty_like(arena.shadow) for _ in range(world)]
dist.all_gather(others, arena.shadow)
same_shadow = all(torch.equal(o, arena.shadow) for o in others)
own = ((arena.data[opt.lo:opt.hi] - data_ref[opt.lo:opt.hi]).abs().max() / (data_ref[opt.lo:opt.hi] - w0[opt.lo:opt.hi]).abs().max()).item()
opt.gather_masters()
torch.cuda.synchronize()
e_masters = ((arena.data - data_ref).norm() / (data_ref - w0).norm()).item()
print(f"[ddp_check] rank {rank}: sharded path: bf16 operand update vs all-reduce+AdamW rel-l2 {e_shadow:.3e}, identical across ranks: {same_shadow}, "
      f"own-slice master max err / max update {own:.3e}, masters after gather rel-l2 of update {e_masters:.3e}, t = {opt.t}", flush=True)
assert e_shadow < 2e-2 and same_shadow and own < 1e-3 and e_masters < 1e-3 and opt.t == 1
shadow_nccl, data_nccl = arena.shadow.clone(), arena.data.clone()

# ---- (3) the same step as ONE kernel over NVLink peer memory (svdx_adamw_step_p2p) vs the NCCL sharded step; then three more steps
# captured in a CUDA graph (fences + kernel replayed) against the eager NCCL optimizer fed the same gradients
arena.data.copy_(w0)
arena.refresh_shadow()
arena.grad.copy_(singles[rank])
torch.cuda.synchronize()
dist.barrier()
popt = P2PShardedAdamW(arena, lr=1e-3, weight_decay=1e-2)
popt.step()
torch.cuda.synchronize()
dist.barrier()
same_as_nccl = torch.equal(arena.shadow, shadow_nccl) if world == 2 else ((arena.shadow.float() - shadow_nccl.float()).abs().max().item() < 1e-2 * shadow_nccl.float().abs().max().item())
own_p2p = torch.equal(arena.data[popt.lo:popt.hi], data_nccl[popt.lo:popt.hi]) if world == 2 else True
others = [torch.empty_like(arena.shadow) for _ in range(world)]
dist.all_gather(others, arena.shadow)
same_ranks = all(torch.equal(o, arena.shadow) for o in others)
print(f"[ddp_check] rank {rank}: p2p fused step: bf16 operands equal to the NCCL sharded step: {same_as_nccl}, own masters equal: {own_p2p}, "
      f"identical across ranks: {same_ranks}, t = {popt.t}", flush=True)
assert same_as_nccl and own_p2p and same_ranks and popt.t == 1
# graph replays: state (m, v, step count) continues from the eager step above; the reference continues the NCCL optimizer
side = torch.cuda.Stream()
side.wait_stream(torch.cuda.current_stream())
g = torch.cuda.CUDAGraph()
snap = [t.clone() for t in (arena.data, arena.shadow, popt.m, popt.v, popt.state)]
with torch.cuda.stream(side):
    popt.step()                      # warm-up outside capture (NCCL communicator on this stream)
torch.cuda.current_stream().wait_stream(side)
torch.cuda.synchronize()
for t, s_ in zip((arena.data, arena.shadow, popt.m, popt.v, popt.state), snap):
    t.copy_(s_)
torch.cuda.synchronize()
dist.barrier()
with torch.cuda.graph(g):
    popt.step()
for t, s_ in zip((arena.data, arena.shadow, popt.m, popt.v, popt.state), snap):
    t.copy_(s_)                       # capture does not run the kernels, but keep the state explicit
torch.cuda.synchronize()
dist.barrier()
for _ in range(3):
    arena.grad.copy_(singles[rank])
    g.replay()
torch.cuda.synchronize()
dist.barrier()
shadow_p2p3 = arena.shadow.clone()
# reference: NCCL sharded optimizer from the same post-step-1 state, three more steps
arena.data.copy_(data_nccl)
arena.shadow.copy_(shadow_nccl)
for _ in range(3):
    arena.grad.copy_(singles[rank])
    opt.step()
torch.cuda.synchronize()
rep_equal = torch.equal(shadow_p2p3, arena.shadow) if world == 2 else ((shadow_p2p3.float() - arena.shadow.float()).abs().max().item() < 1e-2 * arena.shadow.float().abs().max().item())
print(f"[ddp_check] rank {rank}: p2p fused step, 3 CUDA-graph replays vs 3 NCCL sharded steps: operands equal: {rep_equal}, t = {popt.t} / {opt.t}", flush=True)
assert rep_equal and popt.t == 4 and opt.t == 4
# ---- (4) checkpoint and resume of the sharded optimizer. Every rank feeds step t the gradient singles[rank] * (1 + t / 4), so
# the mean gradient is the same at every world size; the weights are "saved" as the gathered masters.
def train(o, a, ts, grad_of):
    for t in ts:
        o.lr = 1e-3 / (1 + 0.1 * t)
        a.grad.copy_(grad_of(t)[:a.numel])
        o.step()
    torch.cuda.synchronize()


own = lambda t: singles[rank] * (1.0 + 0.25 * t)
unet4, arena4 = build()
opt4 = ShardedAdamW(arena4, lr=1e-3, weight_decay=1e-2)
train(opt4, arena4, range(3), own)
sd = opt4.state_dict()                                                  # collective: the same full dict on every rank
opt4.gather_masters()
w3 = arena4.data.clone()
train(opt4, arena4, range(3, 6), own)
opt4.gather_masters()
torch.cuda.synchronize()
w6, m6 = arena4.data.clone(), opt4.m.clone()
arena4.data.copy_(w3)
arena4.refresh_shadow()
opt5 = ShardedAdamW(arena4, lr=7.0, betas=(0.5, 0.5))                   # hyperparameters come from the dict
opt5.load_state_dict(sd)
train(opt5, arena4, range(3, 6), own)
opt5.gather_masters()
torch.cuda.synchronize()
resumed_equal = torch.equal(arena4.data, w6) and torch.equal(opt5.m, m6) and opt5.t == 6
print(f"[ddp_check] rank {rank}: checkpoint at world {world}: resumed run equals the uninterrupted one bit for bit: {resumed_equal}", flush=True)
assert resumed_equal
half = world // 2
sub = dist.new_group(list(range(half))) if half else None
if half and rank < half:
    _, arena_h = build(pad_world=half)
    arena_h.data.copy_(w3[:arena_h.numel])
    arena_h.refresh_shadow()
    opt_h = ShardedAdamW(arena_h, lr=7.0, group=sub)
    assert opt_h.world == half
    opt_h.load_state_dict(sd)
    # sub-rank r stands for ranks r, r + half, ...: their gradients summed and scaled so that the mean over the half world is
    # the mean over the full one
    fold = lambda t: sum(singles[j] for j in range(rank, world, half)) * (half / world) * (1.0 + 0.25 * t)
    train(opt_h, arena_h, range(3, 6), fold)
    opt_h.gather_masters()
    torch.cuda.synchronize()
    e_half = ((arena_h.data - w6[:arena_h.numel]).norm() / (w6 - w3).norm()).item()
    print(f"[ddp_check] rank {rank}: checkpoint of world {world} resumed at world {half}: masters vs the world-{world} continuation, "
          f"rel-l2 of the update {e_half:.3e}, t = {opt_h.t}", flush=True)
    assert e_half < 1e-3 and opt_h.t == 6
elif not half:
    print(f"[ddp_check] rank {rank}: world 1: no smaller world to resume at", flush=True)
# ---- (5) the sharded 8-bit forms against FusedAdamW8bit on the rank-order sum of the gradients. Every rank draws every rank's
# seeded gradients, so each can form the sum in rank order.
def grads8(a, r, t):
    g = torch.Generator(device=dev).manual_seed(1000 * t + r)
    out = torch.zeros_like(a.grad)
    for p in a.params:
        o = a.offset_of[p]
        out[o:o + p.numel()] = torch.randn(p.numel(), generator=g, device=dev) * 1e-2
    return out


for cls in (P2PShardedAdamW8bit, ShardedAdamW8bit):
    _, a_ref = build(block=256)
    _, a8 = build(block=256)
    ref8 = FusedAdamW8bit(a_ref, lr=1e-3, weight_decay=1e-2, min_8bit_size=1024)
    o8 = cls(a8, lr=1e-3, weight_decay=1e-2, min_8bit_size=1024)
    w8 = a8.data.clone()
    for t in range(3):
        ref8.lr = o8.lr = 1e-3 / (1 + t)
        gs = [grads8(a8, r, t) for r in range(world)]
        total = torch.zeros_like(a8.grad)
        for x in gs:
            total += x
        a_ref.grad.copy_(total)
        a8.grad.copy_(gs[rank])
        ref8.step(1.0 / world)
        o8.step()
    torch.cuda.synchronize()
    lo, hi = o8.lo, o8.hi
    if cls is P2PShardedAdamW8bit:
        ok_own = torch.equal(a8.data[lo:hi], a_ref.data[lo:hi])
    else:
        ok_own = ((a8.data[lo:hi] - a_ref.data[lo:hi]).norm() / (a_ref.data[lo:hi] - w8[lo:hi]).norm()).item() < 1e-3
    others = [torch.empty_like(a8.shadow) for _ in range(world)]
    dist.all_gather(others, a8.shadow)
    same8 = all(torch.equal(o, a8.shadow) for o in others)
    sd8, sdr = o8.state_dict(), ref8.state_dict()
    sd_equal = all(torch.equal(v, sdr["state"][i][k]) if isinstance(v, torch.Tensor) else v == sdr["state"][i][k]
                   for i in sdr["state"] for k, v in sd8["state"][i].items())
    exact = cls is P2PShardedAdamW8bit
    print(f"[ddp_check] rank {rank}: {cls.__name__}: own masters vs FusedAdamW8bit on the rank-order sum "
          f"({'bit for bit' if exact else 'rel-l2 of the update < 1e-3'}): {ok_own}, operands identical across ranks: {same8}, "
          f"state_dict equal to FusedAdamW8bit's: {sd_equal if exact else 'not compared (other summation order)'}, t = {o8.t}", flush=True)
    assert ok_own and same8 and o8.t == 3 and (sd_equal or not exact)
dist.barrier()
torch.cuda.synchronize()
sys.stdout.flush()
os._exit(0)      # destroy_process_group() blocks while a CUDA graph that captured NCCL kernels is alive
dist.barrier()
dist.destroy_process_group()
