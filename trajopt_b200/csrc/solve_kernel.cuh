// The whole trust-region SQP of a batch in ONE persistent launch (sco::BasicTrustRegionSQP::optimize(),
// trajopt_sco/src/optimizers.cpp:699-991, for B independent trajectories).
//
// grid = one CTA per SM.  A CTA claims a trajectory, runs `quantum` SQP steps of it back to back — QP subproblem
// (qp_cta_kernel.cuh) then evaluation + convexification + trust-region decision (eval_kernel.cuh), both as device
// functions over the same dynamic shared memory — and hands it back.  Trajectories never interact, so there is no
// grid-wide barrier: a trajectory is never held up by the others' QPs (the lock-step launch pair it replaces
// made every trajectory wait for the slowest QP of each round).  The one exception is opt-in: with group_stop, a seed
// that converges ends its group's siblings at their next iteration top (stopped_at_iteration_top below).
//
// Which trajectory next: the batch is as slow as its longest trajectory (10x the mean; DESIGN.md section 7), and
// what makes a trajectory long is slow ADMM convergence of its QPs, which shows from its first QPs on.  So the
// ready trajectory with the highest mean ADMM iterations per QP so far runs first (not yet started ones before
// all others): the long ones start early and run almost without interruption while the short ones fill the
// remaining SMs.  An event-driven simulation on the per-QP iteration counts of configs[2] puts this order ahead of
// round robin and of lock-step launches, and close to the bound set by the longest trajectory alone.
//
// Hand-over between CTAs goes through sched_state[b] (0 ready, 1 running, 2 finished): release = barrier, fence,
// atomic store by thread 0; acquire = atomic CAS by thread 0, fence, barrier.
#pragma once
#include "eval_kernel.cuh"
#include "qp_cta_kernel.cuh"

namespace tb200 {

enum SolveMode { SOLVE_FULL = 0, SOLVE_QP_ONLY = 1 };
struct SolveCtl {
  int mode, quantum;
  // SOLVE_QP_ONLY (tb200_qp_solve_batch): one Model::optimize() per trajectory on the QP convexified at x_override
  const double* x_override;
  const double* trust_override;
  int* admm_iters_out;
  int* polish_out;
  // SOLVE_FULL
  int* sched_state;             // [B]
  unsigned long long* timers;   // [0..3]: ns in QP steps, ns in evaluation steps, evaluation steps, claims; [4] first
                                // claim (ns, min over CTAs); [8 + b] finish time of trajectory b; [8 + B + b] its busy ns
};

__device__ __forceinline__ unsigned long long global_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}

// The ready trajectory with the highest priority, claimed for this CTA; -1 when none is ready (whatever is still
// running belongs to a CTA that will look again after its quantum).
__device__ inline int claim_trajectory(const DevProblem& p, int* state, int tid) {
  __shared__ unsigned long long s_best[kQpThreads / 32];
  __shared__ int s_pick;
  const unsigned rot = (blockIdx.x * 7u) % static_cast<unsigned>(p.B);  // ties: every CTA prefers a different one
  for (;;) {
    unsigned long long best = 0ull;
    for (int b = tid; b < p.B; b += kQpThreads) {
      if (*reinterpret_cast<volatile int*>(state + b) != 0) continue;
      const int nq = *reinterpret_cast<volatile int*>(p.n_qp_solves + b);
      const int ni = *reinterpret_cast<volatile int*>(p.n_admm_iters + b);
      const float pr = nq ? static_cast<float>(ni) / static_cast<float>(nq) + 1.0f : 3.0e38f;
      const unsigned tie = 0xffffffffu - ((static_cast<unsigned>(b) + p.B - rot) % static_cast<unsigned>(p.B));
      const unsigned long long key = (static_cast<unsigned long long>(__float_as_uint(pr)) << 32) | tie;
      best = key > best ? key : best;
    }
    for (int o = 16; o > 0; o >>= 1) {
      const unsigned long long other = __shfl_xor_sync(0xffffffffu, best, o);
      best = other > best ? other : best;
    }
    if ((tid & 31) == 0) s_best[tid >> 5] = best;
    __syncthreads();
    if (tid == 0) {
      unsigned long long m = 0ull;
      for (int w = 0; w < kQpThreads / 32; ++w) m = s_best[w] > m ? s_best[w] : m;
      int pick = -1;
      if (m != 0ull) {
        const unsigned k = 0xffffffffu - static_cast<unsigned>(m & 0xffffffffull);
        const int b = static_cast<int>((k + rot) % static_cast<unsigned>(p.B));
        pick = (atomicCAS(state + b, 0, 1) == 0) ? b : -2;  // -2: someone else was faster, look again
        if (pick >= 0) __threadfence();
      }
      s_pick = pick;
    }
    __syncthreads();
    const int pick = s_pick;
    __syncthreads();
    if (pick != -2) return pick;
  }
}

__device__ __forceinline__ int load_acquire(const int* a) {
  int v;
  asm volatile("ld.acquire.gpu.global.b32 %0, [%1];" : "=r"(v) : "l"(a) : "memory");
  return v;
}

// Ending a trajectory from outside its own SQP.  Checked where the reference checks its time limit, at the top of every
// SQP iteration (iter = 1 of each merit round and every ++iter, never on a trust-region or QP-failure retry); on the
// device that is just before the QP that begins the iteration.  Two rules, the clock first:
//  1. sco's time limit (optimizers.cpp:738-753): the batch clock is past the trajectory's own max_time (time spent waiting
//     for a CTA counts);
//  2. the group rule (group_stop): a sibling seed of the trajectory's group ended OPT_CONVERGED by its own SQP; the
//     decision step of eval_kernel.cuh set group_done[g] with a release, read here with an acquire.
// Either way the trajectory ends as the reference ends an optimisation from outside: with its last accepted iterate,
// OPT_CONVERGED when its constraints are within its cnt_tolerance (or it has none), else OPT_TIME_LIMIT; ended_by[b] says
// which rule applied.  A QP already running is not interrupted.  Returns (to every thread) whether the trajectory ended.
__device__ inline bool stopped_at_iteration_top(const DevProblem& p, const EvalExtra& ex, const int b, const int tid,
                                                const bool timed) {
  __shared__ int s_stop;
  if (tid == 0) {
    int stop = 0;
    if (p.sqp_top[b] && p.status[b] == 5) {
      if (timed && static_cast<double>(global_ns() - *p.clock_start) * 1e-9 > ex.sqp[b].max_time) stop = 1;
      else if (p.group_stop && load_acquire(p.group_done + b / p.group_size)) stop = 2;
      if (stop) {
        const double* kv = p.cnt_viols + static_cast<size_t>(b) * p.n_cnts;
        double mx = -1e300;
        for (int i = 0; i < p.n_cnts; ++i) mx = fmax(mx, kv[i]);
        p.status[b] = (p.n_cnts == 0 || mx < ex.sqp[b].cnt_tolerance) ? 0 : 3;  // OPT_CONVERGED | OPT_TIME_LIMIT
        p.ended_by[b] = stop;
        atomicSub(p.active_count, 1);
      }
    }
    s_stop = stop;
  }
  __syncthreads();
  return s_stop != 0;  // (thread 0 writes it again only after the barriers of the next QP and evaluation steps)
}
constexpr double kNoTimeLimit = 1.7976931348623157e308;  // DBL_MAX, tb200_default_sqp_params

// SING: the instance for problems with AvoidSingularity objects (solve_inst_<D>_<PAIR>_sing.cu)
template <int DD, int PAIR, int SING = 0>
__global__ void __launch_bounds__(kQpThreads, 1)
solve_kernel(const __grid_constant__ DevProblem p, const __grid_constant__ EvalExtra ex, const __grid_constant__ SolveCtl ctl) {
  const int tid = threadIdx.x;
  const bool qp_only = ctl.mode == SOLVE_QP_ONLY;  // kernel-level entry point: one QP step per trajectory, no scheduler
  const bool timed = !qp_only && ex.sqp_timed;  // (a row with DBL_MAX or NaN never fires)
  const bool stop_checks = timed || (!qp_only && p.group_stop);   // neither: one uniform branch per step
  for (int round = 0;; ++round) {
    const int bq = static_cast<int>(blockIdx.x) + round * static_cast<int>(gridDim.x);
    const int b = qp_only ? (bq < p.B ? bq : -1) : claim_trajectory(p, ctl.sched_state, tid);
    if (b < 0) return;
    unsigned long long t_qp = 0ull, t_ev = 0ull, n_ev = 0ull;
    bool finished = false;
    for (int step = 0; step < ctl.quantum && !finished; ++step) {
      if (stop_checks && stopped_at_iteration_top(p, ex, b, tid, timed)) {
        finished = true;
        break;
      }
      const unsigned long long t0 = global_ns();
      // (a single call site: the QP solve stays inlined in the kernel, as tuned)
      qp_step<DD, PAIR, SING>(p, b, ctl.x_override, ctl.trust_override, ctl.admm_iters_out, ctl.polish_out);
      if (qp_only) break;
      __syncthreads();
      const unsigned long long t1 = global_ns();
      eval_step<DD, SING>(p, ex, EVAL_STEP, b, nullptr);
      __syncthreads();
      const unsigned long long t2 = global_ns();
      t_qp += t1 - t0;
      t_ev += t2 - t1;
      n_ev += 1ull;
      finished = p.status[b] != 5;
    }
    if (qp_only) {
      __syncthreads();
      continue;
    }
    if (tid == 0) {
      if (!qp_only) {  // diagnostics of the schedule (scripts/sched_report.py)
        const unsigned long long now = global_ns();
        atomicMin(ctl.timers + 4, now - t_qp - t_ev);
        ctl.timers[8 + p.B + b] += t_qp + t_ev;
        if (finished) ctl.timers[8 + b] = now;
      }
      atomicAdd(ctl.timers + 0, t_qp);
      atomicAdd(ctl.timers + 1, t_ev);
      atomicAdd(ctl.timers + 2, n_ev);
      atomicAdd(ctl.timers + 3, 1ull);
      __threadfence();
      atomicExch(ctl.sched_state + b, finished ? 2 : 0);
    }
    __syncthreads();
  }
}

}  // namespace tb200
