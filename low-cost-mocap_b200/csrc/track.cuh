// Drone tracking after locate_objects: the reference's KalmanFilter.predict_location (KalmanFilter.py:50-100) and its
// three LowPassFilters per drone (LowPassFilter.py), as step code both the kernels (track.cu) and the g++ build
// (tests/hostcheck/track_host.cpp) run.  Written against geom.cuh only (no CUDA headers).
//
// One call of predict_location is one frame-set with one timestamp t:
//   dt = t - prev_time, prev_time = t (also when no drone is present).  Then for each drone d with at least one object
//   of droneIndex d (in locate_objects order):
//   - T(dt): dt and 0.5 dt^2 blocks, formed in double and rounded to float32;
//   - init: if all 9 entries of the state are 0, its position becomes the FIRST candidate;
//   - predict: x = T x, P = T P T' + 1e-2 I (float32 results of double sums, as cv2's float gemm);
//   - associate: the candidate nearest (double distance, first minimum) to the predicted position;
//   - measure: z = (p, v), p = float32(candidate), v = (p - prev_pos) / dt in float32 -- in double and then rounded
//     while prev_pos is still the reference's integer zero list (before the first measurement and after reset());
//   - correct with H = [I6 0], R = I6: the gain is solved in double from the float32 covariance;
//   - output x[0:6]: the reference returns statePre, which after its init step shares its buffer with statePost, so
//     this is the POSTERIOR.
//   The low-pass outputs are computed afterwards (k_track_lowpass): the k-th call of a drone's filters returns the last
//   output of lfilter(b, a) from zero state over the last L_k samples (track_window).
// Floating point goes through explicit round-to-nearest operations (no contraction, no approximate division or sqrt),
// so the host build and the device give the same bits.
#pragma once
#include "geom.cuh"

#define TRACK_MAX_DRONES 8
#define TRACK_HIST 299                 // samples a drone's filters need from before the current one
#define TRACK_CHANNELS 4               // low-pass inputs per drone: vx, vy, vz, heading

#if defined(__CUDA_ARCH__)
#define TDIV(a, b) __ddiv_rn((a), (b))
#define TSQRT(a) __dsqrt_rn(a)
#define TF32(a) __double2float_rn(a)
#define FSUB(a, b) __fsub_rn((a), (b))
#define FDIV(a, b) __fdiv_rn((a), (b))
#else
#define TDIV(a, b) ((a) / (b))
#define TSQRT(a) sqrt(a)
#define TF32(a) ((float)(a))
#define FSUB(a, b) ((a) - (b))
#define FDIV(a, b) ((a) / (b))
#endif

// scipy.signal.butter(5, 20 / 30): cutoff 20 Hz at the reference's nominal 60 Hz (LowPassFilter.py:13)
#define TRACK_LP_B { 0x1.52c97af6a5633p-3, 0x1.a77bd9b44ebc0p-1, 0x1.a77bd9b44ebc0p+0, 0x1.a77bd9b44ebc0p+0, \
                     0x1.a77bd9b44ebc0p-1, 0x1.52c97af6a5633p-3 }
#define TRACK_LP_A { 0x1.0000000000000p+0, 0x1.a514d17964fd0p+0, 0x1.962c69a214ae5p+0, 0x1.9c197ace69b42p-1, \
                     0x1.d6ef90757fd20p-3, 0x1.be80524dc3515p-6 }

// Persistent state of one drone.  x, P: the cv2 filter's state and errorCovPost; prev_pos / prev_int: the reference's
// prev_positions entry and whether it is still its integer zero list.  k: call index of the drone's low-pass filters
// (kept in 1 .. 450, which gives the same windows); hist_len: samples in its history rows.
struct TrackDrone {
    float  x[9];
    float  P[81];
    float  prev_pos[3];
    int    prev_int;
    int    k;
    int    hist_len;
    double prev_time;
};

// per-step scratch of one drone (shared memory of its warp on the device)
struct TrackWork {
    float x[9], xn[9], P[81], A[81], Ppre[81], gain[54], z[6];
};

// window of the k-th call (k >= 1): the buffer grows to 300 samples, is cut to its last 150 after the 300th, and so on
GEOM_HD int track_window(int k) { return k <= 300 ? k : 151 + (k - 301) % 150; }
GEOM_HD int track_next_call(int k) { return k < 450 ? k + 1 : 301; }

// last output of lfilter(b, a, x[0:L]) from zero state: scipy's transposed direct form, unfused
GEOM_HD double track_lowpass(const double* x, int L) {
    const double b[6] = TRACK_LP_B, a[6] = TRACK_LP_A;
    double z0 = 0.0, z1 = 0.0, z2 = 0.0, z3 = 0.0, z4 = 0.0, y = 0.0;
    for (int n = 0; n < L; ++n) {
        const double xn = x[n];
        y = DADD(z0, DMUL(b[0], xn));
        z0 = DSUB(DADD(z1, DMUL(xn, b[1])), DMUL(y, a[1]));
        z1 = DSUB(DADD(z2, DMUL(xn, b[2])), DMUL(y, a[2]));
        z2 = DSUB(DADD(z3, DMUL(xn, b[3])), DMUL(y, a[3]));
        z3 = DSUB(DADD(z4, DMUL(xn, b[4])), DMUL(y, a[4]));
        z4 = DSUB(DMUL(xn, b[5]), DMUL(y, a[5]));
    }
    return y;
}

// entry (i, j) of the transition matrix; fdt = float32(dt), fh = float32(0.5 dt^2)
GEOM_HD float track_T(int i, int j, float fdt, float fh) {
    if (i == j) return 1.0f;
    if (j == i + 3 && i < 6) return fdt;
    if (j == i + 6 && i < 3) return fh;
    return 0.0f;
}

GEOM_HD void track_dt_terms(double dt, float& fdt, float& fh) {
    fdt = TF32(dt);
    fh = TF32(DMUL(0.5, DMUL(dt, dt)));
}

// the statePost == 0 test of the init step; cand: the first candidate's position
GEOM_HD void track_init(TrackWork& W, const double* cand) {
    bool zero = true;
    for (int i = 0; i < 9; ++i) zero = zero && W.x[i] == 0.0f;
    if (zero)
        for (int i = 0; i < 3; ++i) W.x[i] = TF32(cand[i]);
}

// predict, first half: A = T P, xn = T x (entries lane, lane + nl, ...)
GEOM_HD void track_predict_a(TrackWork& W, float fdt, float fh, int lane, int nl) {
    for (int e = lane; e < 81; e += nl) {
        const int i = e / 9, j = e - 9 * (e / 9);
        double s = 0.0;
        for (int k = 0; k < 9; ++k) s = DADD(s, DMUL((double)track_T(i, k, fdt, fh), (double)W.P[9 * k + j]));
        W.A[e] = TF32(s);
    }
    for (int i = lane; i < 9; i += nl) {
        double s = 0.0;
        for (int k = 0; k < 9; ++k) s = DADD(s, DMUL((double)track_T(i, k, fdt, fh), (double)W.x[k]));
        W.xn[i] = TF32(s);
    }
}

// predict, second half: Ppre = A T' + Q, x = xn
GEOM_HD void track_predict_b(TrackWork& W, float fdt, float fh, int lane, int nl) {
    for (int e = lane; e < 81; e += nl) {
        const int i = e / 9, j = e - 9 * (e / 9);
        double s = 0.0;
        for (int k = 0; k < 9; ++k) s = DADD(s, DMUL((double)W.A[9 * i + k], (double)track_T(j, k, fdt, fh)));
        W.Ppre[e] = TF32(DADD(s, i == j ? (double)1e-2f : 0.0));
    }
    for (int i = lane; i < 9; i += nl) W.x[i] = W.xn[i];
}

// distance of a candidate to the predicted position (np.sqrt(np.sum((p - pred)**2)) in double)
GEOM_HD double track_dist(const double* cand, const float* pred) {
    const double dx = DSUB(cand[0], (double)pred[0]), dy = DSUB(cand[1], (double)pred[1]), dz = DSUB(cand[2], (double)pred[2]);
    return TSQRT(DADD(DADD(DMUL(dx, dx), DMUL(dy, dy)), DMUL(dz, dz)));
}

// the measurement of the chosen candidate; updates the drone's prev_pos
GEOM_HD void track_measure(TrackWork& W, TrackDrone& D, const double* cand, double dt) {
    const float fdt = TF32(dt);
    for (int i = 0; i < 3; ++i) {
        const float p = TF32(cand[i]);
        W.z[i] = p;
        W.z[3 + i] = D.prev_int ? TF32(TDIV((double)p, dt)) : FDIV(FSUB(p, D.prev_pos[i]), fdt);
        D.prev_pos[i] = p;
    }
    D.prev_int = 0;
}

// row r of the gain (r = lane, lane + nl, ... < 9): solves (Ppre[0:6,0:6] + I) g = Ppre[0:6, r] in double
GEOM_HD void track_gain(TrackWork& W, int lane, int nl) {
    for (int r = lane; r < 9; r += nl) {
        double a[6][6], g[6];
        for (int i = 0; i < 6; ++i) {
            for (int j = 0; j < 6; ++j) a[i][j] = (double)TF32(DADD((double)W.Ppre[9 * i + j], i == j ? 1.0 : 0.0));
            g[i] = (double)W.Ppre[9 * i + r];
        }
        for (int c = 0; c < 6; ++c)
            for (int i = c + 1; i < 6; ++i) {
                const double f = TDIV(a[i][c], a[c][c]);
                for (int j = c + 1; j < 6; ++j) a[i][j] = DSUB(a[i][j], DMUL(f, a[c][j]));
                g[i] = DSUB(g[i], DMUL(f, g[c]));
            }
        for (int i = 5; i >= 0; --i) {
            double s = g[i];
            for (int j = i + 1; j < 6; ++j) s = DSUB(s, DMUL(a[i][j], g[j]));
            g[i] = TDIV(s, a[i][i]);
        }
        for (int j = 0; j < 6; ++j) W.gain[6 * r + j] = TF32(g[j]);
    }
}

// correct: xn = x + gain (z - x[0:6]), P = Ppre - gain Ppre[0:6, :]
GEOM_HD void track_correct(TrackWork& W, int lane, int nl) {
    for (int i = lane; i < 9; i += nl) {
        double s = 0.0;
        for (int j = 0; j < 6; ++j) s = DADD(s, DMUL((double)W.gain[6 * i + j], (double)TF32(DSUB((double)W.z[j], (double)W.x[j]))));
        W.xn[i] = TF32(DADD(s, (double)W.x[i]));
    }
    for (int e = lane; e < 81; e += nl) {
        const int i = e / 9, j = e - 9 * (e / 9);
        double s = 0.0;
        for (int k = 0; k < 6; ++k) s = DADD(s, DMUL((double)W.gain[6 * i + k], (double)W.Ppre[9 * k + j]));
        W.P[e] = TF32(DSUB((double)W.Ppre[e], s));
    }
}

GEOM_HD void track_reset(TrackDrone& D, double prev_time) {
    for (int i = 0; i < 9; ++i) D.x[i] = 0.0f;
    for (int i = 0; i < 3; ++i) D.prev_pos[i] = 0.0f;
    D.prev_int = 1;
    D.prev_time = prev_time;
}
