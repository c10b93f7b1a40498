// head_train_emul.cpp -- TEST INFRASTRUCTURE.  Runs csrc/head_train.cuh (the persistent cooperative training kernel of the
// adaptive head) ON THE CPU through tests/cpu_shim/cuda_shim.h: every CUDA thread is a fiber, __syncthreads / shuffles /
// grid barriers are real barriers and the scheduler shuffles the thread order between barriers, so a missing barrier or a
// wrong ownership index changes the result.  The kernel header is compiled as is (it is plain SIMT C++); the result of
// several optimizer steps is compared with a straightforward restatement of the same arithmetic (natural loop order) below.
//   usage: head_train_emul D H0 H1 C n batch G loss(0 ce|1 bce) dropout_p ewc(0|1) update(0|1) seed [z_shift]
//   z_shift: the output biases are moved to +z_shift / -z_shift (even / odd classes) -- saturated logits
#include "cuda_shim.h"
#define AC_CPU_SHIM 1
static inline uint8_t *shim_dyn_smem() { return shim::g_cur->blk->dyn_smem; }
#include "../../adaptive_classifier_b200/csrc/head_train.cuh"

using namespace ac::ht;

struct Host {
    int D, H0, H1, C;
    std::vector<float> W[3], b[3];
};
static void fill(std::vector<float> &v, size_t n, std::mt19937 &rng, float scale) {
    std::uniform_real_distribution<float> u(-1.f, 1.f);
    v.resize(n);
    for (auto &x : v) x = u(rng) * scale;
}

// restatement: one optimizer step (or gradient) in natural order, float arithmetic
struct RefState {
    Host th, m, v, g;
};
static float ref_step(RefState &S, const std::vector<float> &X, const std::vector<int64_t> &yi, const std::vector<float> &yf,
                      const std::vector<int64_t> &rows, int loss_kind, float p_drop, unsigned long long seed, int step, bool ewc,
                      const Host &F, const Host &St, float lam, int C_old, bool update, float *norm_out, float *pen_out) {
    const Host &T = S.th;
    const int D = T.D, H0 = T.H0, H1 = T.H1, C = T.C, B = static_cast<int>(rows.size());
    std::vector<float> h0(B * H0), f0(B * H0), h1(B * H1), f1(B * H1), z(B * C), dz(B * C);
    for (int b = 0; b < B; ++b)
        for (int j = 0; j < H0; ++j) {
            float s = 0.f;
            for (int k = 0; k < D; ++k) s += X[rows[b] * D + k] * T.W[0][j * D + k];
            s += T.b[0][j];
            const float mk = p_drop > 0.f ? ht_mask(p_drop, seed, 2ull * step, static_cast<unsigned long long>(b) * H0 + j) : 1.f;
            h0[b * H0 + j] = (s > 0.f ? s : 0.f) * mk;
            f0[b * H0 + j] = s > 0.f ? mk : 0.f;
        }
    for (int b = 0; b < B; ++b)
        for (int j = 0; j < H1; ++j) {
            float s = 0.f;
            for (int k = 0; k < H0; ++k) s += h0[b * H0 + k] * T.W[1][j * H0 + k];
            s += T.b[1][j];
            const float mk = p_drop > 0.f ? ht_mask(p_drop, seed, 2ull * step + 1, static_cast<unsigned long long>(b) * H1 + j) : 1.f;
            h1[b * H1 + j] = (s > 0.f ? s : 0.f) * mk;
            f1[b * H1 + j] = s > 0.f ? mk : 0.f;
        }
    float loss = 0.f;
    for (int b = 0; b < B; ++b) {
        for (int c = 0; c < C; ++c) {
            float s = 0.f;
            for (int k = 0; k < H1; ++k) s += h1[b * H1 + k] * T.W[2][c * H1 + k];
            z[b * C + c] = s + T.b[2][c];
        }
        if (loss_kind == 0) {
            float mx = -1e30f, sum = 0.f;
            for (int c = 0; c < C; ++c) mx = fmaxf(mx, z[b * C + c]);
            for (int c = 0; c < C; ++c) sum += expf(z[b * C + c] - mx);
            const int64_t y = yi[rows[b]];
            loss += (mx + logf(sum)) - z[b * C + y];
            for (int c = 0; c < C; ++c) dz[b * C + c] = (expf(z[b * C + c] - mx) / sum - (c == y ? 1.f : 0.f)) / B;
        } else {
            float l = 0.f;
            for (int c = 0; c < C; ++c) {
                const float s = 1.f / (1.f + expf(-z[b * C + c])), y = yf[rows[b] * C + c];
                l -= y * fmaxf(logf(s), -100.f) + (1.f - y) * fmaxf(logf(1.f - s), -100.f);
                dz[b * C + c] = (s - y) / fmaxf((1.f - s) * s, 1e-12f) / (static_cast<float>(B) * C) * (1.f - s) * s;
            }
            loss += l / C;
        }
    }
    loss /= B;
    Host &G = S.g;
    std::vector<float> da1(B * H1), da0(B * H0);
    for (int c = 0; c < C; ++c) {
        float sb = 0.f;
        for (int b = 0; b < B; ++b) sb += dz[b * C + c];
        G.b[2][c] = sb;
        for (int k = 0; k < H1; ++k) {
            float s = 0.f;
            for (int b = 0; b < B; ++b) s += dz[b * C + c] * h1[b * H1 + k];
            G.W[2][c * H1 + k] = s;
        }
    }
    for (int b = 0; b < B; ++b)
        for (int k = 0; k < H1; ++k) {
            float s = 0.f;
            for (int c = 0; c < C; ++c) s += dz[b * C + c] * T.W[2][c * H1 + k];
            da1[b * H1 + k] = s * f1[b * H1 + k];
        }
    for (int j = 0; j < H1; ++j) {
        float sb = 0.f;
        for (int b = 0; b < B; ++b) sb += da1[b * H1 + j];
        G.b[1][j] = sb;
        for (int k = 0; k < H0; ++k) {
            float s = 0.f;
            for (int b = 0; b < B; ++b) s += da1[b * H1 + j] * h0[b * H0 + k];
            G.W[1][j * H0 + k] = s;
        }
    }
    for (int b = 0; b < B; ++b)
        for (int k = 0; k < H0; ++k) {
            float s = 0.f;
            for (int j = 0; j < H1; ++j) s += da1[b * H1 + j] * T.W[1][j * H0 + k];
            da0[b * H0 + k] = s * f0[b * H0 + k];
        }
    for (int j = 0; j < H0; ++j) {
        float sb = 0.f;
        for (int b = 0; b < B; ++b) sb += da0[b * H0 + j];
        G.b[0][j] = sb;
        for (int k = 0; k < D; ++k) {
            float s = 0.f;
            for (int b = 0; b < B; ++b) s += da0[b * H0 + j] * X[rows[b] * D + k];
            G.W[0][j * D + k] = s;
        }
    }
    double pen = 0.0;
    if (ewc) {
        const int rows_l[3] = {H0, H1, C_old > 0 && C_old < C ? C_old : C}, K[3] = {D, H0, H1};
        for (int l = 0; l < 3; ++l) {
            for (int i = 0; i < rows_l[l] * K[l]; ++i) {
                const float d = T.W[l][i] - St.W[l][i];
                G.W[l][i] += 2.f * lam / B * F.W[l][i] * d;
                pen += static_cast<double>(F.W[l][i]) * d * d;
            }
            for (int i = 0; i < rows_l[l]; ++i) {
                const float d = T.b[l][i] - St.b[l][i];
                G.b[l][i] += 2.f * lam / B * F.b[l][i] * d;
                pen += static_cast<double>(F.b[l][i]) * d * d;
            }
        }
    }
    double ss = 0.0;
    for (int l = 0; l < 3; ++l) {
        for (float x : G.W[l]) ss += static_cast<double>(x) * x;
        for (float x : G.b[l]) ss += static_cast<double>(x) * x;
    }
    const float norm = static_cast<float>(sqrt(ss));
    *norm_out = norm;
    *pen_out = ewc ? static_cast<float>(lam / B * pen) : 0.f;
    if (update) {
        float coef = 1.f / (norm + 1e-6f);
        coef = coef < 1.f ? coef : 1.f;
        const float lr = 1e-3f, b1 = 0.9f, b2 = 0.999f, eps = 1e-8f, wd = 0.01f;
        const float bc1 = static_cast<float>(1.0 - pow(0.9, step)), bc2s = static_cast<float>(sqrt(1.0 - pow(static_cast<double>(b2), step)));
        auto upd = [&](std::vector<float> &th, std::vector<float> &m, std::vector<float> &v, const std::vector<float> &g) {
            for (size_t i = 0; i < th.size(); ++i) {
                const float gv = g[i] * coef;
                float p = th[i] * (1.f - lr * wd);
                m[i] = m[i] * b1 + gv * (1.f - b1);
                v[i] = v[i] * b2 + gv * gv * (1.f - b2);
                p = p - (lr / bc1) * (m[i] / (sqrtf(v[i]) / bc2s + eps));
                th[i] = p;
            }
        };
        for (int l = 0; l < 3; ++l) { upd(S.th.W[l], S.m.W[l], S.v.W[l], G.W[l]); upd(S.th.b[l], S.m.b[l], S.v.b[l], G.b[l]); }
    }
    return loss;
}

static float max_rel(const std::vector<float> &a, const std::vector<float> &b) {
    float m = 0.f, scale = 1e-6f;
    for (size_t i = 0; i < a.size(); ++i) scale = fmaxf(scale, fabsf(b[i]));
    for (size_t i = 0; i < a.size(); ++i) m = fmaxf(m, fabsf(a[i] - b[i]));
    return m / scale;
}

int main(int argc, char **argv) {
    if (argc < 13) { fprintf(stderr, "usage: D H0 H1 C n batch G loss dropout ewc update seed\n"); return 2; }
    const int D = atoi(argv[1]), H0 = atoi(argv[2]), H1 = atoi(argv[3]), C = atoi(argv[4]), n = atoi(argv[5]), batch = atoi(argv[6]);
    const int G = atoi(argv[7]), loss_kind = atoi(argv[8]);
    const float p_drop = static_cast<float>(atof(argv[9]));
    const bool ewc = atoi(argv[10]) != 0, update = atoi(argv[11]) != 0;
    const unsigned seed = static_cast<unsigned>(atoi(argv[12]));
    const float z_shift = argc > 13 ? static_cast<float>(atof(argv[13])) : 0.f;
    std::mt19937 rng(seed);
    Host T{D, H0, H1, C, {}, {}}, F = T, St = T;
    const int rows[3] = {H0, H1, C}, K[3] = {D, H0, H1};
    for (int l = 0; l < 3; ++l) {
        fill(T.W[l], size_t(rows[l]) * K[l], rng, 0.3f); fill(T.b[l], rows[l], rng, 0.1f);
        fill(F.W[l], size_t(rows[l]) * K[l], rng, 1.f); fill(F.b[l], rows[l], rng, 1.f);
        for (auto &x : F.W[l]) x = fabsf(x);
        for (auto &x : F.b[l]) x = fabsf(x);
        St.W[l] = T.W[l]; St.b[l] = T.b[l];
        for (auto &x : St.W[l]) x += 0.05f;
        for (auto &x : St.b[l]) x -= 0.03f;
    }
    for (int c = 0; c < C; ++c) T.b[2][c] += (c % 2 ? -z_shift : z_shift);
    std::vector<float> X, yf;
    fill(X, size_t(n) * D, rng, 1.f);
    std::vector<int64_t> yi(n), perm(n);
    for (int i = 0; i < n; ++i) { yi[i] = rng() % C; perm[i] = i; }
    std::shuffle(perm.begin(), perm.end(), rng);
    yf.resize(size_t(n) * C);
    for (auto &x : yf) x = (rng() % 3 == 0) ? 1.f : 0.f;
    const int C_old = ewc && C > 2 ? C - 2 : 0;
    const int n_steps = update ? (n + batch - 1) / batch : 1;
    const int n_use = update ? n : (n < batch ? n : batch);

    // ---------------- kernel under the shim
    Host K_th = T, K_m = T, K_v = T, K_g = T, K_q = T;
    for (int l = 0; l < 3; ++l) {
        std::fill(K_m.W[l].begin(), K_m.W[l].end(), 0.f); std::fill(K_m.b[l].begin(), K_m.b[l].end(), 0.f);
        std::fill(K_v.W[l].begin(), K_v.W[l].end(), 0.f); std::fill(K_v.b[l].begin(), K_v.b[l].end(), 0.f);
        std::fill(K_q.W[l].begin(), K_q.W[l].end(), 0.5f); std::fill(K_q.b[l].begin(), K_q.b[l].end(), 0.5f);
    }
    Args a{};
    a.X = X.data(); a.targets = loss_kind == 0 ? static_cast<const void *>(yi.data()) : static_cast<const void *>(yf.data());
    a.perm = update ? perm.data() : nullptr; a.n = n_use; a.batch = batch; a.n_steps = n_steps; a.first_step = update ? 3 : 1;
    for (int l = 0; l < 3; ++l) {
        Layer &L = a.L[l];
        L.W = K_th.W[l].data(); L.b = K_th.b[l].data(); L.rows = rows[l]; L.K = K[l]; L.ewc_rows = rows[l];
        L.mW = K_m.W[l].data(); L.mb = K_m.b[l].data(); L.vW = K_v.W[l].data(); L.vb = K_v.b[l].data();
        L.fW = F.W[l].data(); L.fb = F.b[l].data(); L.sW = St.W[l].data(); L.sb = St.b[l].data();
        L.gW = K_g.W[l].data(); L.gb = K_g.b[l].data(); L.qW = K_q.W[l].data(); L.qb = K_q.b[l].data();
    }
    ht_assign(a, G);
    a.res_mv = seed % 2;                                          // both homes of the AdamW moments
    if (C_old) a.L[2].ewc_rows = C_old;
    a.nst = 2 + static_cast<int>(seed % 6);                       // ring depth 2 .. 7
    a.lr = 1e-3f; a.beta1 = 0.9f; a.beta2 = 0.999f; a.eps = 1e-8f; a.wd = 0.01f; a.max_norm = 1.f; a.dropout_p = p_drop;
    a.loss_kind = loss_kind; a.seed = 11; a.use_ewc = ewc; a.ewc_lambda = 100.f; a.update = update; a.fisher_scale = 0.25f;
    std::vector<float> h0d(size_t(batch) * H0), h1d(size_t(batch) * H1), z(size_t(batch) * C), dz(size_t(batch) * ((C + 3) & ~3), -7.f), da1(size_t(batch) * H1),
        rowloss(batch), part(256), pen(256), stats(3 * n_steps), accum(1, 0.f);
    std::vector<unsigned> bar(4, 0);
    a.h0d = h0d.data(); a.h1d = h1d.data(); a.z = z.data(); a.dz = dz.data(); a.da1 = da1.data(); a.rowloss = rowloss.data();
    a.part = part.data(); a.pen = pen.data(); a.stats = stats.data(); a.loss_accum = accum.data(); a.bar = bar.data();
    const Smem sm = ht_smem_layout(a);
    if (size_t(sm.total) * 4 > 1024 * 1024) { fprintf(stderr, "shared memory %d floats exceeds the shim's 1 MB\n", sm.total); return 2; }
    shim::launch_cooperative(dim3(G), dim3(HT_THREADS), [&] { head_train_kernel(a); }, seed);

    // ---------------- restatement
    RefState S{T, T, T, T};
    for (int l = 0; l < 3; ++l) {
        std::fill(S.m.W[l].begin(), S.m.W[l].end(), 0.f); std::fill(S.m.b[l].begin(), S.m.b[l].end(), 0.f);
        std::fill(S.v.W[l].begin(), S.v.W[l].end(), 0.f); std::fill(S.v.b[l].begin(), S.v.b[l].end(), 0.f);
    }
    float worst = 0.f;
    for (int t = 0; t < n_steps; ++t) {
        std::vector<int64_t> rws;
        for (int b = t * batch; b < n_use && b < (t + 1) * batch; ++b) rws.push_back(update ? perm[b] : b);
        float norm = 0.f, penalty = 0.f;
        const float loss = ref_step(S, X, yi, yf, rws, loss_kind, p_drop, 11, a.first_step + t, ewc, F, St, 100.f, C_old, update, &norm, &penalty);
        const float e0 = fabsf(loss - stats[3 * t]) / fmaxf(1.f, fabsf(loss)), e1 = fabsf(penalty - stats[3 * t + 1]) / fmaxf(1.f, fabsf(penalty)),
                    e2 = fabsf(norm - stats[3 * t + 2]) / fmaxf(1e-3f, fabsf(norm));
        printf("step %d: loss %.6f (kernel %.6f)  penalty %.5f (%.5f)  norm %.6f (%.6f)\n", t, loss, stats[3 * t], penalty, stats[3 * t + 1], norm,
               stats[3 * t + 2]);
        worst = fmaxf(worst, fmaxf(e0, fmaxf(e1, e2)));
    }
    for (int l = 0; l < 3; ++l) {
        if (update) {
            worst = fmaxf(worst, max_rel(K_th.W[l], S.th.W[l])); worst = fmaxf(worst, max_rel(K_th.b[l], S.th.b[l]));
            worst = fmaxf(worst, max_rel(K_m.W[l], S.m.W[l])); worst = fmaxf(worst, max_rel(K_v.W[l], S.v.W[l]));
            worst = fmaxf(worst, max_rel(K_m.b[l], S.m.b[l])); worst = fmaxf(worst, max_rel(K_v.b[l], S.v.b[l]));
        } else {
            worst = fmaxf(worst, max_rel(K_g.W[l], S.g.W[l])); worst = fmaxf(worst, max_rel(K_g.b[l], S.g.b[l]));
            std::vector<float> q(S.g.W[l].size()), qb(S.g.b[l].size());
            for (size_t i = 0; i < q.size(); ++i) q[i] = 0.5f + S.g.W[l][i] * S.g.W[l][i] * 0.25f;
            for (size_t i = 0; i < qb.size(); ++i) qb[i] = 0.5f + S.g.b[l][i] * S.g.b[l][i] * 0.25f;
            worst = fmaxf(worst, max_rel(K_q.W[l], q)); worst = fmaxf(worst, max_rel(K_q.b[l], qb));
        }
    }
    printf("worst relative deviation %.3e -> %s\n", worst, worst < 2e-5f ? "MATCH" : "MISMATCH");
    return worst < 2e-5f ? 0 : 1;
}
