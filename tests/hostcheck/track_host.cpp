// Test-only host build of csrc/track.cuh (the drone tracker's step code), so that the tracker can be checked against
// the oracle on a machine without a GPU.  It walks a batch the way k_track_scan and k_track_lowpass do, one drone and
// one frame-set at a time.  NOT part of libmocap_b200.so and never used by the product path.
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <vector>
#include "../../low-cost-mocap_b200/csrc/track.cuh"

struct HostTracker {
    int D;
    TrackDrone st[TRACK_MAX_DRONES];
    std::vector<double> hist[TRACK_MAX_DRONES][TRACK_CHANNELS];   // every low-pass input so far
};

extern "C" {
void* hc_track_new(int D) {
    HostTracker* h = new HostTracker();
    h->D = D;
    memset(h->st, 0, sizeof(h->st));
    for (int d = 0; d < D; ++d) h->st[d].prev_int = 1;
    return h;
}

void hc_track_free(void* p) { delete static_cast<HostTracker*>(p); }

void hc_track_reset(void* p, double prev_time) {
    HostTracker* h = static_cast<HostTracker*>(p);
    for (int d = 0; d < h->D; ++d) track_reset(h->st[d], prev_time);
}

// the inputs and outputs of mocap_track_objects_dev, host arrays
void hc_track(void* p, const double* objects, const int32_t* drone_index, const int32_t* n_objects, int M, const double* ts,
              int B, float* pos, float* vel, double* heading, uint8_t* present, int32_t* chosen) {
    HostTracker* h = static_cast<HostTracker*>(p);
    const int D = h->D;
    TrackWork W;
    for (int d = 0; d < D; ++d) {
        TrackDrone& S = h->st[d];
        memcpy(W.x, S.x, sizeof(W.x));
        memcpy(W.P, S.P, sizeof(W.P));
        for (int s = 0; s < B; ++s) {
            const double dt = ts[s] - S.prev_time;
            S.prev_time = ts[s];
            const int n = n_objects[s] < 0 ? 0 : n_objects[s] > M ? M : n_objects[s];
            const double* obj = objects + (size_t)s * M * 5;
            const int32_t* di = drone_index + (size_t)s * M;
            const size_t o = (size_t)s * D + d;
            int first = -1;
            for (int j = 0; j < n && first < 0; ++j)
                if (di[j] == d) first = j;
            if (first < 0) {
                for (int i = 0; i < 3; ++i) pos[3 * o + i] = vel[3 * o + i] = 0.0f;
                heading[o] = 0.0;
                present[o] = 0;
                chosen[o] = -1;
                continue;
            }
            track_init(W, obj + (size_t)first * 5);
            float fdt, fh;
            track_dt_terms(dt, fdt, fh);
            track_predict_a(W, fdt, fh, 0, 1);
            track_predict_b(W, fdt, fh, 0, 1);
            double best = INFINITY;
            int bj = first;
            for (int j = first; j < n; ++j)
                if (di[j] == d) {
                    const double dist = track_dist(obj + (size_t)j * 5, W.x);
                    if (dist < best) { best = dist; bj = j; }
                }
            const double* cand = obj + (size_t)bj * 5;
            track_measure(W, S, cand, dt);
            track_gain(W, 0, 1);
            track_correct(W, 0, 1);
            memcpy(W.x, W.xn, sizeof(W.x));
            for (int i = 0; i < 3; ++i) pos[3 * o + i] = W.x[i];
            for (int i = 0; i < 3; ++i) h->hist[d][i].push_back((double)W.x[3 + i]);
            h->hist[d][3].push_back(cand[3]);
            S.k = track_next_call(S.k);
            const int L = track_window(S.k);
            for (int ch = 0; ch < TRACK_CHANNELS; ++ch) {
                const std::vector<double>& row = h->hist[d][ch];
                const double y = track_lowpass(row.data() + row.size() - L, L);
                if (ch < 3) vel[3 * o + ch] = (float)y;
                else heading[o] = y;
            }
            present[o] = 1;
            chosen[o] = bj;
        }
        memcpy(S.x, W.x, sizeof(W.x));
        memcpy(S.P, W.P, sizeof(W.P));
    }
}

// the low-pass filter alone: last output over x[0:L]
double hc_lowpass(const double* x, int L) { return track_lowpass(x, L); }
int hc_window(int k) { return track_window(k); }
int hc_next_call(int k) { return track_next_call(k); }
void hc_lowpass_coefs(double* b, double* a) {
    const double bb[6] = TRACK_LP_B, aa[6] = TRACK_LP_A;
    memcpy(b, bb, sizeof(bb));
    memcpy(a, aa, sizeof(aa));
}
}
