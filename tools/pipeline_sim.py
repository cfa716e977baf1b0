"""Randomised-schedule replay of the plane-gather producer / consumer pipelines with mbarrier PARITY-wait semantics (host
only, no GPU).  A parity wait tells "completed an odd / even number of times", so a waiter must see EVERY phase of a
barrier it waits on.  The replay (random interleavings, overwrite / wrong-data / deadlock detection) shows which role
assignments are sound for `k_wgrad_pl` (and, without the gout ring, `k_conv_pl`):
  * producers: warp w fills unit slots w, w + Wu, ... — sound iff Wu divides `stages` (each warp then owns fixed stages);
  * consumers (the kernels): nc warpgroups each consume EVERY slot in order; a stage is free once all nc have arrived
    (`every=True`) — sound for any nc;
  * Wg warps fill the gout tiles, warp i the row tiles i, i + Wg, ... (Wg divides the ring, so each owns fixed buffers).
With `lag=True` a consumer keeps one wgmma group in flight: it releases slot n - 1 (and, after a row tile's last unit,
that tile's gout buffer) only once it has taken slot n, and releases its last slot at the end.  `k_conv_pl` does this and
maps onto the replay with W = sa producer warps, its weight ring as the gout ring (`gbufs` = its depth sb, 2 or 3) and
its T tiles per weight slice as the units.  In `k_conv_tc` all 8 gather warps fill every slot and each waits on every
slot's "empty" barrier in order; a slot is full once the last of them has arrived, so each behaves as the single
producer Wu = 1 of the replay.
The weight-gradient consumers lag the same way, over a unit ring of `stages` and a gout ring of `gbufs` (2 to 4)
buffers.  In `k_wgrad_pl` Wg warps fill the gout ring and Wu warps the unit slots; in `k_wgrad_tc` all gather warps walk
one slot sequence, each row tile's gout slot and then its units (`joint=True`).
The earlier kernels split the units over nm MMA issuers instead (issuer m owned units u = m (mod nm), `every=False`),
which is sound only if nm divides both `nunits` and `stages`; the two issuer configurations that hung / corrupted tiles on
the GPU (7 producers on 8 stages with 2 issuers, 4 issuers on 6 stages) still fail here and pin the rule.
    python tools/pipeline_sim.py"""
import random
def passed(cnt, parity): return (cnt & 1) != parity
def sim(Wu, nunits, stages, nm, rts, seed, every=False, lag=False, gbufs=2, joint=False, Wg=1):
    """joint=True: one producer (Wu = 1) fills a row tile's gout buffer and then its unit slots, in one slot sequence,
    as the gather warps of `k_wgrad_tc` do; otherwise Wg warps fill the gout ring (`k_wgrad_pl`: warp i the row tiles
    i, i + Wg, ...; the kernel takes Wg dividing gbufs, so that each warp owns fixed buffers)."""
    assert not joint or Wu == 1
    rnd=random.Random(seed)
    full=[0]*stages; empty=[0]*stages; gfull=[0]*gbufs; gempty=[0]*gbufs; arrived=[0]*stages
    data=[None]*stages   # which ord currently in stage (to detect overwrite-before-consume)
    consumed=set(); err=[]
    total=rts*nunits
    def g_filler(w):
        for rti in range(w, rts, Wg):
            gb=rti%gbufs
            while not passed(gempty[gb], ((rti//gbufs)&1)^1): yield
            gfull[gb]+=1; yield
    def producer(w):
        o=w; st=w; ph=0
        while o<total:
            while not passed(empty[st], ph^1): yield
            if data[st] is not None and data[st] not in consumed: err.append(('overwrite',o,data[st]))
            data[st]=o; full[st]+=1
            o+=Wu; st+=Wu
            if st>=stages: st-=stages; ph^=1
            yield
    def joint_producer():
        st=0; ph=0
        for rti in range(rts):
            gb=rti%gbufs
            while not passed(gempty[gb], ((rti//gbufs)&1)^1): yield
            gfull[gb]+=1; yield
            for u in range(nunits):
                o=rti*nunits+u
                while not passed(empty[st], ph^1): yield
                if data[st] is not None and data[st] not in consumed: err.append(('overwrite',o,data[st]))
                data[st]=o; full[st]+=1
                st+=1
                if st==stages: st=0; ph^=1
                yield
    def release(st, o):
        arrived[st]+=1
        if not every or arrived[st]==nm:   # every=True: the stage is free once all nm consumers arrived
            arrived[st]=0; consumed.add(o); empty[st]+=1
    def release_g(gb):
        gcommit[gb]+=1
        if gcommit[gb]%nm==0: gempty[gb]+=1
    def issuer(m):
        st=0; ph=0
        held=None                          # lag=True: (stage, ord, gout buffer or None) of the slot still in flight
        for git in range(rts):
            gb=git%gbufs
            while not passed(gfull[gb], (git//gbufs)&1): yield
            for u in range(nunits):
                if every or u%nm==m:
                    while not passed(full[st], ph): yield
                    o=git*nunits+u
                    if data[st]!=o: err.append(('wrongdata',o,data[st]))
                    if lag:
                        if held is not None:
                            release(held[0], held[1])
                            if held[2] is not None: release_g(held[2])
                        held=(st, o, gb if u==nunits-1 else None)
                    else:
                        release(st, o)
                st+=1
                if st==stages: st=0; ph^=1
                yield
            if not lag: release_g(gb)
        if held is not None:
            release(held[0], held[1])
            if held[2] is not None: release_g(held[2])
    gcommit=[0]*gbufs
    fillers=[joint_producer()] if joint else [g_filler(w) for w in range(Wg)]+[producer(w) for w in range(Wu)]
    agents=fillers+[issuer(m) for m in range(nm)]
    alive=list(range(len(agents))); idle=0
    while alive:
        i=rnd.choice(alive)
        before=(tuple(full),tuple(empty),tuple(gfull),tuple(gempty),len(consumed))
        for _ in range(rnd.randint(1,8)):
            try: next(agents[i])
            except StopIteration: alive.remove(i); break
        after=(tuple(full),tuple(empty),tuple(gfull),tuple(gempty),len(consumed))
        idle=0 if after!=before else idle+1
        if idle>30000: return 'DEADLOCK'
    return 'ERR' if err else 'ok'
def producer_choice(stages, max_producers=7):
    """The unit-producer count k_wgrad_pl derives from the ring depth: the largest divisor of `stages` <= 7."""
    return max(d for d in range(1, max_producers + 1) if stages % d == 0)


def gout_producer_choice(gbufs, Wu, warps=8):
    """The gout-producer count k_wgrad_pl derives: the largest divisor of the gout ring depth <= the warps left."""
    return max(d for d in range(1, warps - Wu + 1) if gbufs % d == 0)


def host_choice(nunits, stages, max_issuers=4, max_producers=7):
    """Role counts of the earlier multi-issuer kernels (kept to replay the configurations that failed)."""
    Wu = max(d for d in range(1, max_producers + 1) if stages % d == 0)
    nm = 1
    for c in range(2, max_issuers + 1):        # k_wgrad_pl takes any count; k_conv_pl only the powers of two among them
        if nunits % c == 0 and stages % c == 0:
            nm = c
    return Wu, nm


if __name__ == "__main__":
    for stages in range(2, 9):                      # the current kernels: two consumer warpgroups see every slot
        res=[sim(producer_choice(stages),4,stages,2,14,s,every=True) for s in range(40)]
        print("consumers", stages, {k:res.count(k) for k in set(res)})
    for sa in range(3, 9):                          # k_conv_pl, one wgmma group in flight per consumer
        res=[sim(W,t,sa,2,14,s,every=True,lag=True,gbufs=sb) for W in (sa,1) for t in (1,2,4) for sb in (2,3) for s in range(5)]
        print("lagged conv consumers", sa, {k:res.count(k) for k in set(res)})
    for (Wu,nunits,stages,nm) in ((7,8,8,2),(4,8,8,2),(4,8,8,4),(6,8,6,2),(6,6,6,3),(4,4,4,4),(5,4,5,1),(7,7,8,1),(2,2,2,2),(6,8,6,4)):
        res=[sim(Wu,nunits,stages,nm,14,s) for s in range(80)]
        print((Wu,nunits,stages,nm), {k:res.count(k) for k in set(res)})
