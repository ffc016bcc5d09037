"""Multi-GPU calibration: shard independent equalization chains over ranks, exchange the scale vectors once.

SURVEY.md section 8(e).  The unit of parallelism is the *chain* (relations linked first->second are serially dependent
inside a sweep; different chains never touch the same layer).  One process per GPU (torch.distributed; NCCL on the GPUs,
gloo in the CPU tests):

  1. every rank builds the same chain list from `relations` and the same static LPT assignment (by weight elements);
  2. each rank equalizes ITS chains with the persistent kernel (dfq_cle_run) on its own replica of the model;
  3. ONE all_gather_into_tensor of a flat, equal-size-padded fp32 buffer carries the accumulated S of every relation;
  4. every rank replays the S of the chains it does not own on its replica (rows * S, columns * 1/S: dfq_cle_run with
     apply_only), so all ranks finish with the same full model and no weight tensor ever crosses NVLink.

Convergence (dfq.py:81-115 is a GLOBAL rule: sum over all layers):
  mode="per_chain"  each chain stops on its own exit rule (one convergence group per chain).  Differs from the
                    reference only in chains that would have kept iterating because ANOTHER chain had not converged
                    yet; those extra sweeps multiply by s = 1 +- ulp, far inside the 1e-5 contract.  No per-sweep traffic.
  mode="exact"      bit-faithful sweep count: every rank first iterates a scratch copy of its shard recording its
                    per-sweep metric, ONE all_reduce(SUM) of those vectors yields the global metric per sweep, the
                    reference's exit rule is replayed on it, and the shard is then equalized for exactly that many
                    sweeps.  Twice the local work, still a single small collective.

Replaying S (step 4) applies the accumulated product in one multiplication instead of one per sweep: owner ranks hold
bit-exact values, replicas agree to ~3e-6 relative (SURVEY 8e).

Sharded evaluation (DESIGN.md section 3.14): `shard` gives each rank a contiguous block of the dataset, and the
classify, segment and detect evaluators' `all_reduce` merge the ranks' evaluators into the one-process result through
`_gather_rows` below.
"""
from __future__ import annotations

from typing import Dict, List, Sequence, Tuple

import torch
import torch.distributed as dist
import torch.nn as nn

from .engine import Session


def _all_gather_flat(recv: torch.Tensor, send: torch.Tensor, group=None):
    """all_gather_into_tensor; gloo has no CUDA all-gather, so with that backend (the single-GPU multi-process tests) the
    buffers are staged through the host.  NCCL (one process per GPU) takes the device path."""
    if send.is_cuda and dist.get_backend(group) == "gloo":
        r = torch.empty(recv.shape, dtype=recv.dtype)
        dist.all_gather_into_tensor(r, send.cpu(), group=group)
        recv.copy_(r)
    else:
        dist.all_gather_into_tensor(recv, send, group=group)


def _world_rank(group=None) -> Tuple[int, int]:
    if not dist.is_initialized():
        return 1, 0
    return dist.get_world_size(group), dist.get_rank(group)


def shard(n: int, group=None) -> range:
    """This rank's share of a dataset of n items for sharded evaluation: one contiguous block per rank, in rank order, the
    first n % world ranks taking one item more.  A rank may get an empty range.  Without a process group, or with one
    rank, range(n).

    torch.utils.data.DistributedSampler is not a substitute: it deals items to the ranks in turn and pads the last round
    by repeating items, so repeated images are counted twice, and the detection evaluator's order among equal scores (the
    order images were added, DESIGN.md section 4) is no longer the dataset's order.  With shard(), the ranks' blocks
    concatenated in rank order are range(n), which is what the evaluators' all_reduce() relies on."""
    if isinstance(n, bool) or not isinstance(n, int) or n < 0:
        raise ValueError("shard: n must be a non-negative int, got %r" % (n,))
    world, rank = _world_rank(group)
    base, extra = divmod(n, world)
    start = rank * base + min(rank, extra)
    return range(start, start + base + (rank < extra))


def _idle_device() -> torch.device:
    """Where an evaluator that never received a batch stages its (zero) share of a reduction: the current CUDA device."""
    return torch.device("cuda", torch.cuda.current_device())


def _gather_rows(send: torch.Tensor, group=None) -> torch.Tensor:
    """[world, n]: every rank's 1-D `send` (n elements on every rank), in rank order.  One process: send as one row."""
    world, _ = _world_rank(group)
    if world == 1:
        return send.reshape(1, -1).clone()
    recv = torch.empty(world * send.numel(), dtype=send.dtype, device=send.device)
    _all_gather_flat(recv, send.contiguous(), group)
    return recv.view(world, -1)


def build_chains(relations) -> List[List[int]]:
    """Group relation indices into chains (rel j follows rel i when first(j) == second(i)); order inside a chain and
    the order of chains follow the relation list."""
    by_first = {rr.get_idxs()[0]: i for i, rr in enumerate(relations)}
    is_follower = set()
    for rr in relations:
        nxt = by_first.get(rr.get_idxs()[1])
        if nxt is not None:
            is_follower.add(nxt)
    chains = []
    for i, rr in enumerate(relations):
        if i in is_follower:
            continue
        chain, cur = [i], rr
        while cur.get_idxs()[1] in by_first:
            j = by_first[cur.get_idxs()[1]]
            chain.append(j)
            cur = relations[j]
        chains.append(chain)
    return chains


def partition_lpt(costs: Sequence[int], world: int) -> List[int]:
    """Longest-processing-time-first: item i -> rank.  Deterministic (ties by index), identical on every rank."""
    load = [0] * world
    owner = [0] * len(costs)
    for i in sorted(range(len(costs)), key=lambda i: (-costs[i], i)):
        r = min(range(world), key=lambda r: (load[r], r))
        owner[i] = r
        load[r] += costs[i]
    return owner


def _replay_exit_rule(diffs: Sequence[float], converge_thres: float, converge_count: int, state=None):
    """dfq.py:81-115 on a recorded sequence of diff_tmp values -> number of sweeps the reference would run, or None when
    the rule has not fired by the end of the recording.  `state` ([diff, count, sweeps so far]) carries the rule across
    consecutive recordings (the kernel records 64 sweeps per launch)."""
    st = state if state is not None else [10, 0, 0]
    for d in diffs:
        st[2] += 1
        if abs(st[0] - d) > 1e-9:
            st[1], st[0] = 0, d
        else:
            st[1] += 1
        if not (st[0] > converge_thres and st[1] < converge_count):
            return st[2]
    return None


def sharded_cross_layer_equalization(graph, relations, targ_type, s_range=(1e-8, 1e8), converge_thres=2e-7,
                                     converge_count=20, signed=False, eps=0, mode="per_chain", group=None, max_record=64,
                                     replicas="replay"):
    """cross_layer_equalization (dfq.py:78-117) with the chains sharded over the ranks of `group`.
    Every rank must call it with the same graph/relations; every rank's model ends up fully equalized.
    replicas="replay": only the scale vectors are exchanged and every rank replays the S of the chains it does not own
                       (weights within ~3e-6 of the owner's; no weight crosses NVLink - the stack-sized workloads);
    replicas="exact":  the all-gathered buffer ALSO carries the equalized weights / biases / BN vectors of every rank's chains
                       (a real model: a few tens of MB), so every rank ends with bit-identical parameters - what the steps
                       downstream of the equalization need when they are ill-conditioned in the last bit of the weights
                       (bias correction, DESIGN.md section 4) and every rank must reach the same model.
    Returns dict(owner=[rank per chain], sweeps=..., chains=...)."""
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    rank = dist.get_rank(group) if dist.is_initialized() else 0
    with torch.no_grad():
        chains = build_chains(relations)
        cost = []
        for ch in chains:
            keys = {relations[i].get_idxs()[0] for i in ch} | {relations[i].get_idxs()[1] for i in ch}
            cost.append(sum(graph[k].weight.numel() for k in keys))
        owner = partition_lpt(cost, world)

        sess = Session()
        index: Dict[object, int] = {}

        def layer_of(key, need_bias):
            mod = graph[key]
            if need_bias and mod.bias is None:
                mod.bias = nn.Parameter(torch.zeros(mod.weight.size(0), dtype=torch.float32, device=mod.weight.device),
                                        requires_grad=False)
                if key in index:
                    sess.attach_bias(index[key], mod.bias)
            if key not in index:
                index[key] = sess.add_layer(mod.weight, mod.bias)
            return index[key]

        bn_bound = {}
        table = []
        for rr in relations:
            first, second, bn_idx = rr.get_idxs()
            l1, l2 = layer_of(first, True), layer_of(second, False)
            if bn_idx not in bn_bound:
                bn = graph[bn_idx]
                bn_bound[bn_idx] = (sess.bind(bn.fake_weight), sess.bind(bn.fake_bias))
            table.append((l1, l2) + bn_bound[bn_idx])
        sess.upload()

        mine = [i for c, ch in enumerate(chains) if owner[c] == rank for i in ch]
        mine_group = {i: g for g, c in enumerate([c for c in range(len(chains)) if owner[c] == rank]) for i in chains[c]}
        n_rel = len(relations)
        chan = [sess.layer(t[0])["rows"] for t in table]
        slot = max(chan) if chan else 0
        S_all = torch.ones(n_rel, slot, dtype=torch.float32, device=sess.device)
        sweeps = 0
        if mine:
            local = [table[i] for i in mine]
            if mode == "per_chain":
                plan = sess.plan_cle(local, groups=[mine_group[i] for i in mine])
                res = sess.run_cle_plan(plan, s_range, converge_thres, converge_count, signed, eps)
                sweeps = res.n_sweeps
            elif mode == "exact":
                plan = sess.plan_cle(local)
                sess._ensure_room()
                snapshot = sess.arena.clone()
            else:
                raise ValueError(mode)
        else:
            plan = None
        if mode == "exact":
            # Record the shard's metric in launches of `max_record` (<= 64, what DfqCleResult.diffs holds) sweeps that
            # continue from each other, reduce every recording over the ranks and replay the reference's exit rule on the
            # global sequence until it fires - however many sweeps that takes (the kernel's own safety net is 4096).
            max_record = max(1, min(int(max_record), 64))
            rule, sweeps = [10, 0, 0], None
            while sweeps is None:
                local_diffs = torch.zeros(max_record, dtype=torch.float64, device=sess.device)
                if plan is not None:
                    rec = sess.run_cle_plan(plan, s_range, 0.0, 1 << 30, signed, eps, max_sweeps=max_record)
                    local_diffs[:len(rec.diffs)] = torch.tensor(rec.diffs, dtype=torch.float64, device=sess.device)
                if world > 1:
                    dist.all_reduce(local_diffs, group=group)        # the global dfq.py:105-108 metric per sweep
                sweeps = _replay_exit_rule(local_diffs.tolist(), converge_thres, converge_count, rule)
                if sweeps is None and rule[2] >= 4096:
                    raise RuntimeError("sharded equalization: the exit rule of dfq.py:81-115 did not fire within 4096 sweeps "
                                       "(last metric %g)" % rule[0])
            if plan is not None:
                sess.arena.copy_(snapshot)
                sess.run_cle_plan(plan, s_range, 0.0, 1 << 30, signed, eps, max_sweeps=sweeps)
        if plan is not None:
            for i, off in zip(mine, plan["s_offs"]):
                S_all[i, :chan[i]] = sess.view(off, chan[i])

        # ---- the one exchange of the path: all-gather of the scale vectors ------------------------------------------
        if world > 1:
            gathered = torch.empty(world * n_rel * slot, dtype=torch.float32, device=sess.device)
            _all_gather_flat(gathered, S_all.reshape(-1).contiguous(), group)
            gathered = gathered.view(world, n_rel, slot)
            rel_owner = [0] * n_rel
            for c, ch in enumerate(chains):
                for i in ch:
                    rel_owner[i] = owner[c]
            S_all = torch.stack([gathered[rel_owner[i], i] for i in range(n_rel)])
            others = [i for i in range(n_rel) if rel_owner[i] != rank]
            if replicas == "exact":
                # every tensor a chain's equalization writes: weights and biases of its layers, fake_weight / fake_bias of its BNs
                def chain_views(c):
                    seen, out = set(), []
                    for i in chains[c]:
                        l1, l2, obw, obb = table[i]
                        for li in (l1, l2):
                            if li not in seen:
                                seen.add(li)
                                l = sess.layer(li)
                                out.append((l["w_off"], l["rows"] * l["cols"] * l["kk"])); out.append((l["bias_off"], l["rows"]))
                        out.append((obw, chan[i])); out.append((obb, chan[i]))
                    return out
                per_rank = [[v for c in range(len(chains)) if owner[c] == r for v in chain_views(c)] for r in range(world)]
                cap = max(sum(n for _, n in vs) for vs in per_rank)
                send = torch.zeros(cap, dtype=torch.float32, device=sess.device)
                o = 0
                for off, n in per_rank[rank]:
                    send[o:o + n].copy_(sess.view(off, n)); o += n
                recv = torch.empty(world * cap, dtype=torch.float32, device=sess.device)
                _all_gather_flat(recv, send, group)
                for r in range(world):
                    if r == rank:
                        continue
                    o = r * cap
                    for off, n in per_rank[r]:
                        sess.view(off, n).copy_(recv[o:o + n]); o += n
            elif replicas == "replay":
                if others:
                    rplan = sess.plan_cle([table[i] for i in others])
                    for i, off in zip(others, rplan["s_offs"]):
                        sess.view(off, chan[i]).copy_(S_all[i, :chan[i]])
                    sess.run_cle_plan(rplan, s_range, signed=signed, eps=eps, apply_only=True)
            else:
                raise ValueError(replicas)
        sess.download()
        for i, rr in enumerate(relations):
            S = S_all[i, :chan[i]].clone()
            rr.set_scale_vec(S if graph[rr.get_idxs()[0]].weight.is_cuda else S.cpu())
        return dict(owner=owner, chains=chains, sweeps=sweeps)


def sharded_bias_correction(graph, bottoms, targ_type, bits_weight=8, bn_type=torch.nn.BatchNorm2d, signed=False, group=None,
                            replicate_below: int = 1 << 23):
    """bias_correction (dfq.py:173-293) with the heavy part - one pass over every corrected weight - sharded over ranks.

    The recurrence of the pass (a layer's expectation reads the fake_bias the previous corrected layer's -delta landed
    in, dfq.py:204-206,239,293) orders the layers into dependency LEVELS (graphwalk.bias_correction_recipe); layers of one
    level are independent.  Per level:
      * a level with fewer than `replicate_below` weight elements (every level of a serial network such as MobileNetV2) is
        computed by EVERY rank on its replica: the kernel is deterministic, so all ranks hold identical bits and nothing is
        exchanged;
      * a larger level is split over the ranks (LPT by weight elements); ONE all_gather_into_tensor of a padded buffer then
        carries, for every layer of the level, its corrected bias and the updated fake_bias of the BN that follows
        (SURVEY 8(e) "Collective"), and every rank copies in the rows it did not compute.
    Every rank must call it with the same (already equalized) model; every rank's model ends up fully corrected.
    Returns dict(levels=..., sharded_levels=..., owner={layer key: rank})."""
    from .dfq import _zero_bias
    from .graphwalk import bias_correction_recipe
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    rank = dist.get_rank(group) if dist.is_initialized() else 0
    with torch.no_grad():
        recipe = bias_correction_recipe(graph, bottoms, targ_type, bn_type)
        if not recipe:
            return dict(levels=0, sharded_levels=0, owner={})
        sess = Session()
        bn_bound: Dict[object, Tuple[int, int]] = {}

        def bn_offsets(key):
            if key not in bn_bound:
                bn = graph[key]
                bn_bound[key] = (sess.bind(bn.fake_weight), sess.bind(bn.fake_bias))
            return bn_bound[key]

        items = []
        for step in recipe:
            mod = graph[step["layer"]]
            if mod.bias is None:
                _zero_bias(mod)                                       # dfq.py:290-291
            li = sess.add_layer(mod.weight, mod.bias, weight_writeback=False)
            terms = []
            for t in step["terms"]:
                ow, ob = bn_offsets(t["bn"])
                terms.append(dict(bn_w_off=ow, bn_b_off=ob, n=graph[t["bn"]].fake_bias.numel(), relu=t["relu"], op=t["op"]))
            nxt = bn_offsets(step["next_bn"])[1] if step["next_bn"] is not None else -1
            items.append(dict(layer=li, signed=signed, level=0, next_bn_b_off=nxt, terms=terms, key=step["layer"],
                              numel=mod.weight.numel(), rows=mod.weight.size(0), lev=step["level"]))
        levels = sorted({it["lev"] for it in items})
        # ---- plan every launch before the arena is materialised (scratch is part of it) -------------------------------
        schedule, owner_of = [], {}
        for lev in levels:
            its = [it for it in items if it["lev"] == lev]
            shard = world > 1 and len(its) >= 2 and sum(it["numel"] for it in its) >= replicate_below
            if shard:
                own = partition_lpt([it["numel"] for it in its], world)
                mine = [it for it, o in zip(its, own) if o == rank]
            else:
                own, mine = [rank] * len(its), its
            for it, o in zip(its, own):
                owner_of[it["key"]] = o if shard else -1              # -1: replicated
            plan = sess.plan_bias_correct(mine) if mine else None
            schedule.append((its, own, shard, plan))
        sess.upload()
        n_sharded = 0
        for its, own, shard, plan in schedule:
            if plan is not None:
                sess.run_bias_correct_plan(plan, 8)                   # quirk Q2 (dfq.py:218): always 8 bits
            if not shard:
                continue
            n_sharded += 1
            slot = max(it["rows"] for it in its)
            per_rank = [[it for it, o in zip(its, own) if o == r] for r in range(world)]
            cap = max(len(p) for p in per_rank)
            send = torch.zeros(cap, 2, slot, dtype=torch.float32, device=sess.device)
            for k, it in enumerate(per_rank[rank]):
                l = sess.layer(it["layer"])
                send[k, 0, :it["rows"]] = sess.view(l["bias_off"], it["rows"])
                if it["next_bn_b_off"] >= 0:
                    send[k, 1, :it["rows"]] = sess.view(it["next_bn_b_off"], it["rows"])
            recv = torch.empty(world * cap * 2 * slot, dtype=torch.float32, device=sess.device)
            _all_gather_flat(recv, send.reshape(-1), group)
            recv = recv.view(world, cap, 2, slot)
            for r in range(world):
                if r == rank:
                    continue
                for k, it in enumerate(per_rank[r]):
                    l = sess.layer(it["layer"])
                    sess.view(l["bias_off"], it["rows"]).copy_(recv[r, k, 0, :it["rows"]])
                    if it["next_bn_b_off"] >= 0:
                        sess.view(it["next_bn_b_off"], it["rows"]).copy_(recv[r, k, 1, :it["rows"]])
        sess.download()
        return dict(levels=len(levels), sharded_levels=n_sharded, owner=owner_of)


def sync_observers(model: nn.Module, group=None) -> int:
    """Data-parallel `update_quant_range` (improve_dfq.py:280-300): every rank drives its QuantMeasure observers over ITS share
    of the distilled batches in `update_stat` mode (running_max = max(running_max, stat), quantize.py:103-107), then calls
    this once: two all-reduces (MIN over every running_min, MAX over every running_max, 2 floats per observer) leave all
    ranks with the ranges a single process would have reached over all batches - max/min are associative, so the result does
    not depend on how whole batches were dealt to the ranks (SURVEY 8e, "replicas only").  Returns the number of observers."""
    from .utils.quantize import QuantMeasure
    obs = [m for m in model.modules() if isinstance(m, QuantMeasure)]
    if not obs or not dist.is_initialized() or dist.get_world_size(group) == 1:
        return len(obs)
    with torch.no_grad():
        dev = obs[0].running_min.device
        mn = torch.cat([m.running_min.reshape(1).to(dev) for m in obs])
        mx = torch.cat([m.running_max.reshape(1).to(dev) for m in obs])
        dist.all_reduce(mn, op=dist.ReduceOp.MIN, group=group)
        dist.all_reduce(mx, op=dist.ReduceOp.MAX, group=group)
        for i, m in enumerate(obs):
            m.running_min.reshape(1).copy_(mn[i:i + 1])
            m.running_max.reshape(1).copy_(mx[i:i + 1])
    return len(obs)
