// lion_b200 -- device-resident RK45 (Dormand-Prince 5(4)) for the probability-flow ODE of the VPSDE.
//
// A restatement of the integrator the reference runs on the host: scipy's RK45 as solve_ivp(..., t_eval=...) drives it
// through the vendored torchdiffeq scipy_solver wrapper (utils/diffusion_continuous.py:90-249).  Followed files of
// scipy 1.18: integrate/_ivp/rk.py (RungeKutta._step_impl, rk_step, the RK45 tableaux C, A, B, E, P, RkDenseOutput)
// and integrate/_ivp/common.py (select_initial_step, norm).  The state is float64 as scipy's; the model sees the state
// rounded to fp32 and returns fp32, as the wrapper's torch.tensor(y).to(device, float32) and .cpu().numpy() do.
//
// What differs from the host route is only where things run: every scalar lives in LionOdeState on the device, the
// controller is one thread, and the norms reduce fixed-size partials in a fixed order, so a whole step attempt
// (5 stage evaluations, the FSAL evaluation and these kernels) can be captured once and replayed.  Sums over stages are
// evaluated left to right without FMA contraction; numpy's dot may associate differently, so states agree with scipy's
// to rounding, not bit for bit.
#include "common.cuh"
#include "../../include/lion_b200.h"

namespace lion {

constexpr int ODE_NB = 256;      // blocks of every norm pass = partials per sum
constexpr int ODE_NT = 256;

// RK45 tableaux (rk.py), each entry the same float64 quotient Python computes
__constant__ double c_C[7] = {0.0, 1.0 / 5, 3.0 / 10, 4.0 / 5, 8.0 / 9, 1.0, 1.0};
__constant__ double c_A[6][5] = {
    {0, 0, 0, 0, 0},
    {1.0 / 5, 0, 0, 0, 0},
    {3.0 / 40, 9.0 / 40, 0, 0, 0},
    {44.0 / 45, -56.0 / 15, 32.0 / 9, 0, 0},
    {19372.0 / 6561, -25360.0 / 2187, 64448.0 / 6561, -212.0 / 729, 0},
    {9017.0 / 3168, -355.0 / 33, 46732.0 / 5247, 49.0 / 176, -5103.0 / 18656}};
__constant__ double c_B[6] = {35.0 / 384, 0, 500.0 / 1113, 125.0 / 192, -2187.0 / 6784, 11.0 / 84};
__constant__ double c_E[7] = {-71.0 / 57600, 0, 71.0 / 16695, -71.0 / 1920, 17253.0 / 339200, -22.0 / 525, 1.0 / 40};
__constant__ double c_P[7][4] = {
    {1, -8048581381.0 / 2820520608, 8663915743.0 / 2820520608, -12715105075.0 / 11282082432},
    {0, 0, 0, 0},
    {0, 131558114200.0 / 32700410799, -68118460800.0 / 10900136933, 87487479700.0 / 32700410799},
    {0, -1754552775.0 / 470086768, 14199869525.0 / 1410260304, -10690763975.0 / 1880347072},
    {0, 127303824393.0 / 49829197408, -318862633887.0 / 49829197408, 701980252875.0 / 199316789632},
    {0, -282668133.0 / 205662961, 2019193451.0 / 616988883, -1453857185.0 / 822651844},
    {0, 40617522.0 / 29380423, -110615467.0 / 29380423, 69997945.0 / 29380423}};

constexpr double SAFETY = 0.9, MIN_FACTOR = 0.2, MAX_FACTOR = 10.0;
constexpr double ERROR_EXPONENT = -1.0 / (4 + 1);   // -1 / (error_estimator_order + 1)
constexpr double INIT_EXPONENT = 1.0 / (4 + 1);     // 1 / (order + 1) in select_initial_step

__global__ void k_ode_init(LionOdeState* st, const float* __restrict__ y0, double* __restrict__ y, size_t n, double t0,
                           double t_bound, double rtol, double atol, int negate) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) y[i] = (double)y0[i];
  if (i == 0) {
    LionOdeState s = {};
    s.t = t0; s.t_bound = t_bound;
    s.direction = t_bound != t0 ? (t_bound > t0 ? 1.0 : -1.0) : 1.0;     // np.sign(t_bound - t0), 1 for an empty span
    s.rtol = rtol; s.atol = atol;
    s.status = t0 == t_bound ? LION_ODE_DONE : LION_ODE_RUNNING;
    s.negate = negate;
    *st = s;
  }
}

__global__ void k_ode_stage(LionOdeState* st, const double* __restrict__ y, double* __restrict__ y_new,
                            const double* __restrict__ K, size_t n, int stage, float* __restrict__ x,
                            float* __restrict__ t_model, int B) {
  if (st->status != LION_ODE_RUNNING) return;
  const double t = st->t, h = st->h;
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    const double yi = y[i];
    double v;
    if (stage == 0) {
      v = yi;
    } else if (stage == LION_ODE_STAGE_PROBE) {                 // y1 = y0 + h0 * direction * f0
      v = __dadd_rn(yi, __dmul_rn(__dmul_rn(st->h0, st->direction), K[i]));
    } else if (stage < 6) {                                     // y + np.dot(K[:s].T, a[:s]) * h
      double acc = __dmul_rn(K[i], c_A[stage][0]);
      for (int j = 1; j < stage; ++j) acc = __dadd_rn(acc, __dmul_rn(K[(size_t)j * n + i], c_A[stage][j]));
      v = __dadd_rn(yi, __dmul_rn(acc, h));
    } else {                                                    // y_new = y + h * np.dot(K[:-1].T, B)
      double acc = __dmul_rn(K[i], c_B[0]);
      for (int j = 1; j < 6; ++j) acc = __dadd_rn(acc, __dmul_rn(K[(size_t)j * n + i], c_B[j]));
      v = __dadd_rn(yi, __dmul_rn(h, acc));
      y_new[i] = v;
    }
    x[i] = __double2float_rn(v);
  }
  if (blockIdx.x == 0) {
    double ts = stage == LION_ODE_STAGE_PROBE ? __dadd_rn(t, __dmul_rn(st->h0, st->direction))
              : stage == 0 ? t
              : stage == 6 ? __dadd_rn(t, h)                  // fun(t + h, y_new)
              : __dadd_rn(t, __dmul_rn(c_C[stage], h));       // fun(t + c * h, y + dy)
    const float tf = __double2float_rn(st->negate ? -ts : ts);
    for (int b = threadIdx.x; b < B; b += blockDim.x) t_model[b] = tf;
  }
}

// dx/dt = f(t) x + ((0.5 g2(t)) eps) / sqrt(var(t)) with the VPSDE's scalars evaluated as torch does on a 0-dim fp32
// tensor t: every Python float enters as float32(value computed in float64), every operation is rounded on its own.
//   var(t) = 1.0 - (1.0 - sigma2_0) * exp(-beta_start * t - 0.5 * (beta_end - beta_start) * t * t)
//   g2(t)  = beta_start + (beta_end - beta_start) * t,   f(t) = -0.5 * g2(t)
struct VpsdeConsts { float neg_bs, half_db, one_m_s2, db, bs; };
__global__ void k_ode_rhs(LionOdeState* st, const float* __restrict__ x, const float* __restrict__ eps,
                          double* __restrict__ Ks, size_t n, VpsdeConsts c, const float* __restrict__ t_model) {
  if (st->status != LION_ODE_RUNNING) return;
  const float t = t_model[0];
  const float var = __fsub_rn(1.0f, __fmul_rn(c.one_m_s2, expf(__fsub_rn(__fmul_rn(c.neg_bs, t),
                                                                        __fmul_rn(__fmul_rn(c.half_db, t), t)))));
  const float g2 = __fadd_rn(__fmul_rn(c.db, t), c.bs);
  const float f = __fmul_rn(-0.5f, g2);
  const float half_g2 = __fmul_rn(0.5f, g2);
  const float sd = __fsqrt_rn(var);
  const bool neg = st->negate != 0;
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    float d = __fadd_rn(__fmul_rn(f, x[i]), __fdiv_rn(__fmul_rn(half_g2, eps[i]), sd));
    Ks[i] = (double)(neg ? -d : d);
  }
  if (i == 0) st->nfe += 1;
}

__device__ __forceinline__ double ode_scale(const LionOdeState& s, double a) {   // atol + |y| * rtol
  return __dadd_rn(s.atol, __dmul_rn(a, s.rtol));
}

// Sums of squares over fixed-size partials: thread i of block b takes elements b*NT + i, then + NB*NT, ... in order, and
// the block adds its threads' values in a fixed tree.  what = INIT_H0: [0] y / scale, [1] f0 / scale;
// INIT_H1: [0] (f1 - f0) / scale (scale of y0 both times); END: [0] (h * sum_j E_j K_j) / (atol + max(|y|, |y_new|) rtol).
__global__ void __launch_bounds__(ODE_NT) k_ode_norms(const LionOdeState* st, const double* __restrict__ y,
                                                      const double* __restrict__ y_new, const double* __restrict__ K,
                                                      size_t n, int what, double* __restrict__ partials) {
  __shared__ double red[2][ODE_NT];
  const LionOdeState s = *st;
  double a0 = 0.0, a1 = 0.0;
  if (s.status == LION_ODE_RUNNING) {
    for (size_t i = (size_t)blockIdx.x * ODE_NT + threadIdx.x; i < n; i += (size_t)ODE_NB * ODE_NT) {
      if (what == LION_ODE_INIT_H0) {
        const double sc = ode_scale(s, fabs(y[i]));
        const double u = __ddiv_rn(y[i], sc), v = __ddiv_rn(K[i], sc);
        a0 = __dadd_rn(a0, __dmul_rn(u, u));
        a1 = __dadd_rn(a1, __dmul_rn(v, v));
      } else if (what == LION_ODE_INIT_H1) {
        const double sc = ode_scale(s, fabs(y[i]));
        const double u = __ddiv_rn(__dsub_rn(K[n + i], K[i]), sc);
        a0 = __dadd_rn(a0, __dmul_rn(u, u));
      } else {
        double acc = __dmul_rn(K[i], c_E[0]);
        for (int j = 1; j < 7; ++j) acc = __dadd_rn(acc, __dmul_rn(K[(size_t)j * n + i], c_E[j]));
        const double sc = ode_scale(s, fmax(fabs(y[i]), fabs(y_new[i])));
        const double u = __ddiv_rn(__dmul_rn(acc, s.h), sc);
        a0 = __dadd_rn(a0, __dmul_rn(u, u));
      }
    }
  }
  red[0][threadIdx.x] = a0;
  red[1][threadIdx.x] = a1;
  __syncthreads();
  for (int o = ODE_NT / 2; o > 0; o >>= 1) {
    if (threadIdx.x < o) {
      red[0][threadIdx.x] = __dadd_rn(red[0][threadIdx.x], red[0][threadIdx.x + o]);
      red[1][threadIdx.x] = __dadd_rn(red[1][threadIdx.x], red[1][threadIdx.x + o]);
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    partials[blockIdx.x] = red[0][0];
    partials[ODE_NB + blockIdx.x] = red[1][0];
  }
}

__global__ void __launch_bounds__(ODE_NT) k_ode_control(LionOdeState* st, const double* __restrict__ partials, size_t n,
                                                        int what) {
  static_assert(ODE_NB == ODE_NT, "one partial per thread");
  __shared__ double red[2][ODE_NT];
  red[0][threadIdx.x] = partials[threadIdx.x];
  red[1][threadIdx.x] = partials[ODE_NB + threadIdx.x];
  __syncthreads();
  for (int o = ODE_NT / 2; o > 0; o >>= 1) {
    if (threadIdx.x < o) {
      red[0][threadIdx.x] = __dadd_rn(red[0][threadIdx.x], red[0][threadIdx.x + o]);
      red[1][threadIdx.x] = __dadd_rn(red[1][threadIdx.x], red[1][threadIdx.x + o]);
    }
    __syncthreads();
  }
  if (threadIdx.x != 0) return;
  LionOdeState s = *st;
  if (s.status != LION_ODE_RUNNING) return;
  const double rn = sqrt((double)n);                              // x.size ** 0.5
  const double interval = fabs(__dsub_rn(s.t_bound, s.t));
  if (what == LION_ODE_INIT_H0) {
    const double d0 = __ddiv_rn(sqrt(red[0][0]), rn), d1 = __ddiv_rn(sqrt(red[1][0]), rn);
    double h0 = (d0 < 1e-5 || d1 < 1e-5) ? 1e-6 : __ddiv_rn(__dmul_rn(0.01, d0), d1);
    s.h0 = fmin(h0, interval);                                    // h0 = min(h0, interval_length)
    s.d1 = d1;
  } else if (what == LION_ODE_INIT_H1) {
    const double d2 = __ddiv_rn(__ddiv_rn(sqrt(red[0][0]), rn), s.h0);
    const double h1 = (s.d1 <= 1e-15 && d2 <= 1e-15) ? fmax(1e-6, __dmul_rn(s.h0, 1e-3))
                                                     : pow(__ddiv_rn(0.01, fmax(s.d1, d2)), INIT_EXPONENT);
    s.h_abs = fmin(fmin(__dmul_rn(100.0, s.h0), h1), interval);   // min(100 * h0, h1, interval_length, max_step = inf)
    s.new_step = 1;
  } else if (what == LION_ODE_BEGIN) {
    if (s.new_step) {                                             // the start of RungeKutta._step_impl
      s.min_step = __dmul_rn(10.0, fabs(__dsub_rn(nextafter(s.t, s.direction * INFINITY), s.t)));
      if (s.h_abs < s.min_step) s.h_abs = s.min_step;
      s.step_rejected = 0;
      s.new_step = 0;
    }
    s.accepted = 0;
    if (s.h_abs < s.min_step) {
      s.status = LION_ODE_TOO_SMALL;
    } else {
      double h = __dmul_rn(s.h_abs, s.direction);
      double t_new = __dadd_rn(s.t, h);
      if (__dmul_rn(s.direction, __dsub_rn(t_new, s.t_bound)) > 0) t_new = s.t_bound;
      h = __dsub_rn(t_new, s.t);
      s.h = h;
      s.h_abs = fabs(h);
      s.t_new = t_new;
    }
  } else {                                                        // LION_ODE_END
    const double err = __ddiv_rn(sqrt(red[0][0]), rn);
    s.err_norm = err;
    if (err < 1) {
      double factor = err == 0 ? MAX_FACTOR : fmin(MAX_FACTOR, __dmul_rn(SAFETY, pow(err, ERROR_EXPONENT)));
      if (s.step_rejected) factor = fmin(1.0, factor);
      s.h_abs = __dmul_rn(s.h_abs, factor);
      s.t = s.t_new;
      s.n_accepted += 1;
      s.accepted = 1;
      s.new_step = 1;
      if (__dmul_rn(s.direction, __dsub_rn(s.t, s.t_bound)) >= 0) s.status = LION_ODE_DONE;
    } else {
      s.h_abs = __dmul_rn(s.h_abs, fmax(MIN_FACTOR, __dmul_rn(SAFETY, pow(err, ERROR_EXPONENT))));
      s.step_rejected = 1;
      s.n_rejected += 1;
    }
  }
  *st = s;
}

__global__ void k_ode_commit(const LionOdeState* st, double* __restrict__ y, const double* __restrict__ y_new,
                             double* __restrict__ K, size_t n) {
  if (st->status != LION_ODE_RUNNING || !st->accepted) return;
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    y[i] = y_new[i];
    K[i] = K[(size_t)6 * n + i];                                  // FSAL: self.f = f_new
  }
}

// RkDenseOutput at x = 1: y_old + h * (Q . [1, 1, 1, 1]) with Q = K.T . P
__global__ void k_ode_dense_end(const LionOdeState* st, const double* __restrict__ y, const double* __restrict__ K,
                                size_t n, float* __restrict__ out) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (st->n_accepted == 0) { out[i] = __double2float_rn(y[i]); return; }
  double q[4];
  for (int j = 0; j < 4; ++j) {
    double acc = __dmul_rn(K[i], c_P[0][j]);
    for (int s = 1; s < 7; ++s) acc = __dadd_rn(acc, __dmul_rn(K[(size_t)s * n + i], c_P[s][j]));
    q[j] = acc;
  }
  const double qs = __dadd_rn(__dadd_rn(__dadd_rn(q[0], q[1]), q[2]), q[3]);
  out[i] = __double2float_rn(__dadd_rn(__dmul_rn(st->h, qs), y[i]));
}

}  // namespace lion

using namespace lion;

static inline unsigned ode_grid(size_t n) { return (unsigned)cdivz(n, 256); }

extern "C" size_t lion_ode_state_bytes(void) { return sizeof(LionOdeState); }

extern "C" int lion_ode_init(LionOdeState* st, const float* y0, double* y, size_t n, double t0, double t_bound, double rtol,
                             double atol, int negate, void* stream) {
  LION_REQUIRE(st && y0 && y && n > 0 && rtol > 0 && atol >= 0, "lion_ode_init: bad arguments");
  Ctx c;
  c.stream = (cudaStream_t)stream;
  LION_LAUNCH(&c, k_ode_init, ode_grid(n), 256, 0, st, y0, y, n, t0, t_bound, rtol, atol, negate);
  return check_launch(&c, "lion_ode_init");
}

extern "C" int lion_ode_stage(LionOdeState* st, const double* y, double* y_new, const double* K, size_t n, int stage,
                              float* x, float* t_model, int B, void* stream) {
  LION_REQUIRE(st && y && K && x && t_model && n > 0 && B > 0 && (stage != 6 || y_new) &&
               ((stage >= 0 && stage <= 6) || stage == LION_ODE_STAGE_PROBE), "lion_ode_stage: bad arguments");
  Ctx c;
  c.stream = (cudaStream_t)stream;
  LION_LAUNCH(&c, k_ode_stage, ode_grid(n), 256, 0, st, y, y_new, K, n, stage, x, t_model, B);
  return check_launch(&c, "lion_ode_stage");
}

extern "C" int lion_ode_rhs(LionOdeState* st, const float* x, const float* eps, double* K, size_t n, int stage,
                            double beta_start, double beta_end, double sigma2_0, const float* t_model, void* stream) {
  LION_REQUIRE(st && x && eps && K && t_model && n > 0 && ((stage >= 0 && stage <= 6) || stage == LION_ODE_STAGE_PROBE),
               "lion_ode_rhs: bad arguments");
  VpsdeConsts k;
  k.neg_bs = (float)(-beta_start);
  k.half_db = (float)(0.5 * (beta_end - beta_start));
  k.one_m_s2 = (float)(1.0 - sigma2_0);
  k.db = (float)(beta_end - beta_start);
  k.bs = (float)beta_start;
  const int row = stage == LION_ODE_STAGE_PROBE ? 1 : stage;
  Ctx c;
  c.stream = (cudaStream_t)stream;
  LION_LAUNCH(&c, k_ode_rhs, ode_grid(n), 256, 0, st, x, eps, K + (size_t)row * n, n, k, t_model);
  return check_launch(&c, "lion_ode_rhs");
}

extern "C" int lion_ode_norms(const LionOdeState* st, const double* y, const double* y_new, const double* K, size_t n,
                              int what, double* partials, void* stream) {
  LION_REQUIRE(st && y && K && partials && n > 0 && (what != LION_ODE_END || y_new) &&
               (what == LION_ODE_INIT_H0 || what == LION_ODE_INIT_H1 || what == LION_ODE_END), "lion_ode_norms: bad arguments");
  Ctx c;
  c.stream = (cudaStream_t)stream;
  LION_LAUNCH(&c, k_ode_norms, ODE_NB, ODE_NT, 0, st, y, y_new, K, n, what, partials);
  return check_launch(&c, "lion_ode_norms");
}

extern "C" int lion_ode_control(LionOdeState* st, const double* partials, size_t n, int what, void* stream) {
  LION_REQUIRE(st && partials && n > 0 && what >= LION_ODE_INIT_H0 && what <= LION_ODE_BEGIN, "lion_ode_control: bad arguments");
  Ctx c;
  c.stream = (cudaStream_t)stream;
  LION_LAUNCH(&c, k_ode_control, 1, ODE_NT, 0, st, partials, n, what);
  return check_launch(&c, "lion_ode_control");
}

extern "C" int lion_ode_commit(const LionOdeState* st, double* y, const double* y_new, double* K, size_t n, void* stream) {
  LION_REQUIRE(st && y && y_new && K && n > 0, "lion_ode_commit: bad arguments");
  Ctx c;
  c.stream = (cudaStream_t)stream;
  LION_LAUNCH(&c, k_ode_commit, ode_grid(n), 256, 0, st, y, y_new, K, n);
  return check_launch(&c, "lion_ode_commit");
}

extern "C" int lion_ode_dense_end(const LionOdeState* st, const double* y, const double* K, size_t n, float* out, void* stream) {
  LION_REQUIRE(st && y && K && out && n > 0, "lion_ode_dense_end: bad arguments");
  Ctx c;
  c.stream = (cudaStream_t)stream;
  LION_LAUNCH(&c, k_ode_dense_end, ode_grid(n), 256, 0, st, y, K, n, out);
  return check_launch(&c, "lion_ode_dense_end");
}
