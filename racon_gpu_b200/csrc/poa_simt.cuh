/*
 * poa_simt.cuh -- the tiny warp-programming layer the POA engine is written against.
 *
 * The engine (poa_core.cuh) is one-window-per-warp code.  It is written ONCE and compiled in two
 * flavours:
 *   - nvcc (__CUDACC__): the product.  POA_LANES(l) runs its body once with l = this thread's lane,
 *     PerLane<T> is a register, collectives are warp shuffles / ballots.
 *   - g++  (tests/emu only): a lock-step emulation used by the CPU test-suite to check every graph
 *     phase against the oracle without a GPU.  POA_LANES(l) loops l = 0..31, PerLane<T> is an array
 *     of 32 values, collectives are plain loops.  The emulation is test infrastructure; the product
 *     library never contains it.
 *
 * Rules the engine code obeys so both flavours mean the same thing:
 *   - state that must survive from one POA_LANES block to the next lives in PerLane<T> variables
 *     (or in the workspace memory);
 *   - lanes inside one POA_LANES block never read what another lane writes in the same block;
 *   - a POA_SYNC() separates blocks that communicate through memory.
 */
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define POA_FN __device__ __forceinline__
#define POA_FN_NOINLINE __device__ __noinline__
#define POA_DEVICE 1
#else
#define POA_FN static inline
#define POA_FN_NOINLINE static
#define POA_DEVICE 0
#endif

namespace b200poa {

#if POA_DEVICE

template <class T>
struct PerLane {
    T v;
    __device__ __forceinline__ T& operator[](int) { return v; }
    __device__ __forceinline__ const T& operator[](int) const { return v; }
};

#define POA_LANES(l) for (int l = (int)(threadIdx.x & 31u), _poa_once = 1; _poa_once; _poa_once = 0)
#define POA_LANE0 if ((threadIdx.x & 31u) == 0u)
#define POA_SYNC() __syncwarp()
/* Between two phases: what one lane wrote to the workspace (plain, streaming or atomic stores) must be visible to
 * every access path the other lanes use next (cached loads, L1-bypassing asynchronous copies).  In the proven-uniform
 * build __syncwarp() is elided altogether, so the ordering is asked for explicitly, once per phase boundary. */
#define POA_FENCE() __threadfence_block()

/* Warp-uniform control flow and the compiler (ptxas 12.9, sm_90a; tests/test_codegen.py pins it).
 *
 * A warp collective (shuffle, vote, redux, __syncwarp) is one instruction only where ptxas can PROVE that the whole
 * warp arrives together.  As soon as ONE collective of the module sits in control flow it cannot prove uniform, EVERY
 * collective of EVERY function gets a "BRA.DIV -> WARPSYNC.COLLECTIVE" slow path, BSSY/BSYNC brackets and the
 * registers to feed them: +43 % instructions, 14 % fewer windows/s on this kernel.  The engine is one window per warp,
 * so its control flow IS uniform; what it takes to make that provable:
 *   1. Scalars reach a noinline phase function BY VALUE (Params, ReadGeom, lengths).  A value loaded through a
 *      reference parameter lives in local memory and counts as lane-dependent.
 *   2. State that must come back through a reference (WinState) is laundered after the call (winstate_uniform) and
 *      at the function's entry: poa_uniform() = redux.sync, whose result lands in a uniform register (REDUX into a UR).
 *   3. Values read back from a shuffle, from inline-asm memory accesses or from generic-pointer loads are uniform in
 *      fact but not provably: launder them (poa_uniform / poa_uniform_pred = vote) before they steer a loop or a branch
 *      that contains a collective -- the path position in the traceback, the row record in the fill.
 *   4. Never leave a loop or a function from lane-dependent control flow: set a flag, decide by a vote.
 *   5. After a lane-0 block that is followed by a loop back edge, reconverge explicitly (__syncwarp).
 *   6. Keep the number of live uniform values small: derive (edge capacity from node capacity) instead of carrying.
 *   7. No atomicAdd inside a lane-divergent loop (ptxas aggregates it with a match/vote of its own, which sits in
 *      divergent flow by construction): use an idempotent plain store where a flag is all that is asked, or hoist the
 *      atomic into straight-line predicated code (mark_subgraph / topsort_roots).
 * In the proven state __syncwarp() costs no instruction at all and uniform arithmetic moves to the uniform datapath. */
POA_FN int poa_uniform(int x) { return __reduce_max_sync(0xffffffffu, x); }
/* a de-facto uniform predicate made provably uniform by a vote */
POA_FN bool poa_uniform_pred(bool x) { return __any_sync(0xffffffffu, x) != 0; }

/* exclusive prefix sum over lanes, returns the warp total (provably uniform) */
POA_FN int warp_exscan(PerLane<int>& x) {
    const int lane = (int)(threadIdx.x & 31u);
    int v = x.v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        int t = __shfl_up_sync(0xffffffffu, v, d);
        if (lane >= d) v += t;
    }
    const int total = __reduce_add_sync(0xffffffffu, x.v);
    x.v = v - x.v;
    return total;
}
POA_FN unsigned warp_ballot(const PerLane<int>& p) { return __ballot_sync(0xffffffffu, p.v != 0); }
POA_FN int warp_max(const PerLane<int>& x) { return __reduce_max_sync(0xffffffffu, x.v); }
POA_FN int warp_min(const PerLane<int>& x) { return __reduce_min_sync(0xffffffffu, x.v); }
/* value held by lane `src` (src uniform) */
POA_FN int warp_get(const PerLane<int>& x, int src) { return __shfl_sync(0xffffffffu, x.v, src); }
/* make a lane-0 scalar uniform across the warp */
POA_FN int warp_bcast0(int x) { return __reduce_max_sync(0xffffffffu, (threadIdx.x & 31u) == 0u ? x : (int)0x80000000); }
/* out[l] = x[l+1] (lane 31 keeps its own value) */
POA_FN void warp_shift_down1(const PerLane<int>& x, PerLane<int>& out) { out.v = __shfl_down_sync(0xffffffffu, x.v, 1); }
/* inclusive prefix max over lanes, in place */
POA_FN void warp_incl_max(PerLane<int>& x) {
    const int lane = (int)(threadIdx.x & 31u);
    int v = x.v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, v, d);
        if (lane >= d && t > v) v = t;
    }
    x.v = v;
}

/* out[l] = x[l-1] (lane 0 keeps its own value) */
POA_FN void warp_shift_up1(const PerLane<int>& x, PerLane<int>& out) { out.v = __shfl_up_sync(0xffffffffu, x.v, 1); }

#else /* ---------------------------------------------------------------- host emulation */

template <class T>
struct PerLane {
    T v[32];
    T& operator[](int l) { return v[l]; }
    const T& operator[](int l) const { return v[l]; }
};

#define POA_LANES(l) for (int l = 0; l < 32; ++l)
#define POA_LANE0
#define POA_SYNC() ((void)0)
#define POA_FENCE() ((void)0)

POA_FN int warp_exscan(PerLane<int>& x) {
    int run = 0;
    for (int l = 0; l < 32; ++l) {
        int t = x.v[l];
        x.v[l] = run;
        run += t;
    }
    return run;
}
POA_FN unsigned warp_ballot(const PerLane<int>& p) {
    unsigned m = 0;
    for (int l = 0; l < 32; ++l)
        if (p.v[l]) m |= 1u << l;
    return m;
}
POA_FN int warp_max(const PerLane<int>& x) {
    int m = x.v[0];
    for (int l = 1; l < 32; ++l)
        if (x.v[l] > m) m = x.v[l];
    return m;
}
POA_FN int warp_min(const PerLane<int>& x) {
    int m = x.v[0];
    for (int l = 1; l < 32; ++l)
        if (x.v[l] < m) m = x.v[l];
    return m;
}
POA_FN int warp_get(const PerLane<int>& x, int src) { return x.v[src]; }
POA_FN int warp_bcast0(int x) { return x; }
POA_FN int poa_uniform(int x) { return x; }
POA_FN bool poa_uniform_pred(bool x) { return x; }
POA_FN void warp_shift_down1(const PerLane<int>& x, PerLane<int>& out) {
    for (int l = 0; l < 31; ++l) out.v[l] = x.v[l + 1];
    out.v[31] = x.v[31];
}
POA_FN void warp_incl_max(PerLane<int>& x) {
    for (int l = 1; l < 32; ++l)
        if (x.v[l - 1] > x.v[l]) x.v[l] = x.v[l - 1];
}
POA_FN void warp_shift_up1(const PerLane<int>& x, PerLane<int>& out) {
    for (int l = 31; l > 0; --l) out.v[l] = x.v[l - 1];
    out.v[0] = x.v[0];
}

#endif

POA_FN int poa_popc(unsigned m) {
#if POA_DEVICE
    return __popc(m);
#else
    return __builtin_popcount(m);
#endif
}
POA_FN int poa_ffs(unsigned m) { /* index of lowest set bit, m != 0 */
#if POA_DEVICE
    return __ffs((int)m) - 1;
#else
    return __builtin_ctz(m);
#endif
}

} // namespace b200poa
