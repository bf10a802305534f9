// Host-side emulation of the generic real FFT of deepfilternet_b200/csrc/dfb_fft_generic.cuh: runs the Stockham stages
// (every butterfly of a stage, then the next stage, as the CTA does between its barriers), the split step of the forward
// and the merge step of the inverse transform in fp32 on the CPU, and checks both against a double-precision DFT with
// the element-wise bound of tests/test_gpu_stft_sizes.py (fft_rounds):
//   |err| <= gamma(n) * sum |inputs|   (forward: the real frame; inverse: the Hermitian spectrum, inner bins twice)
// Prints the worst err / bound over every size and exits non-zero when it exceeds 1.  Built and run by
// tests/test_stft_sizes_host.py (no GPU needed).
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "../../deepfilternet_b200/csrc/dfb_fft_generic.cuh"
using namespace dfb;

static const double U = 1.0 / 16777216.0;

// roundings along one input -> output path (same table as fft_rounds in tests/test_gpu_stft_sizes.py)
static int fft_rounds(const GenFftPlan &pl) {
    int n = pl.N % 2 == 0 ? 4 : 0;
    for (int s = 0; s < pl.nst; s++) {
        const int R = pl.rad[s];
        n += 6 + (R == 2 ? 1 : R == 4 ? 2 : R == 3 ? 4 : R == 5 ? 6 : R == 7 ? 8 : R + 1);
    }
    return n;
}

// the M-point complex transform of buf (in place, result in buf)
template <bool INV>
static void cfft(const GenFftPlan &pl, const float2 *tw, std::vector<float2> &buf) {
    std::vector<float2> other(pl.M);
    float2 *src = buf.data(), *dst = other.data();
    int Ns = 1;
    for (int s = 0; s < pl.nst; s++) {
        const int R = pl.rad[s];
        for (int j = 0; j < pl.M / R; j++) gen_stage_bfly<INV>(src, dst, pl.M, Ns, R, j, tw, pl.N / pl.M);
        Ns *= R;
        float2 *t = src; src = dst; dst = t;
    }
    if (src != buf.data()) for (int i = 0; i < pl.M; i++) buf[i] = src[i];
}

// returns max err / bound of forward and inverse at size N
static double check(int N) {
    GenFftPlan pl;
    std::vector<float2> tw;
    if (!gen_fft_plan(N, pl, tw)) { printf("N=%d: no plan\n", N); return 1e30; }
    const int M = pl.M, F = N / 2 + 1;
    const double g = fft_rounds(pl) * U / (1.0 - fft_rounds(pl) * U);
    std::vector<float> x(N);
    for (auto &v : x) v = (float)(rand() / (double)RAND_MAX - 0.5);
    // forward
    std::vector<float2> buf(M);
    if (N % 2 == 0) for (int n = 0; n < M; n++) buf[n] = make_float2(x[2 * n], x[2 * n + 1]);
    else for (int n = 0; n < M; n++) buf[n] = make_float2(x[n], 0.f);
    cfft<false>(pl, tw.data(), buf);
    std::vector<float2> X(F);
    if (N % 2 == 0) {
        for (int k = 0; k <= M / 2; k++) {
            float2 xk, xnk;
            rfft_split(buf[k], buf[(M - k) % M], tw[k], xk, xnk);
            X[k] = xk;
            X[M - k] = xnk;
        }
    } else {
        for (int k = 0; k < F; k++) X[k] = buf[k];
    }
    double l1 = 0;
    for (float v : x) l1 += fabs(v);
    double worst = 0;
    for (int k = 0; k < F; k++) {
        double ar = 0, ai = 0;
        for (int n = 0; n < N; n++) {
            const double a = -2.0 * M_PI * (double)((long)k * n % N) / N;
            ar += x[n] * cos(a); ai += x[n] * sin(a);
        }
        worst = fmax(worst, hypot(ar - X[k].x, ai - X[k].y) / (g * l1));
    }
    // inverse from a random Hermitian half spectrum (imaginary parts of DC and, for even N, Nyquist ignored)
    for (auto &v : X) v = make_float2((float)(rand() / (double)RAND_MAX - 0.5), (float)(rand() / (double)RAND_MAX - 0.5));
    X[0].y = 0.f;
    if (N % 2 == 0) X[F - 1].y = 0.f;
    if (N % 2 == 0) {
        for (int k = 0; k <= M / 2; k++) {
            const float2 w = tw[k];
            float2 zk, znk;
            irfft_merge(X[k], X[M - k], make_float2(w.x, -w.y), zk, znk);
            buf[k] = zk;
            if (k > 0 && k < M - k) buf[M - k] = znk;
        }
    } else {
        buf[0] = X[0];
        for (int k = 1; k < F; k++) { buf[k] = X[k]; buf[N - k] = cconj(X[k]); }
    }
    cfft<true>(pl, tw.data(), buf);
    double hl1 = 0;
    for (int k = 0; k < F; k++) hl1 += (k == 0 || (N % 2 == 0 && k == F - 1) ? 1.0 : 2.0) * hypot(X[k].x, X[k].y);
    for (int n = 0; n < N; n++) {
        double y = 0;
        for (int k = 0; k < F; k++) {
            const double a = 2.0 * M_PI * (double)((long)k * n % N) / N;
            const double h = (k == 0 || (N % 2 == 0 && k == F - 1)) ? 1.0 : 2.0;
            y += h * (X[k].x * cos(a) - X[k].y * sin(a));
        }
        const float got = N % 2 == 0 ? (n % 2 == 0 ? buf[n / 2].x : buf[n / 2].y) : buf[n].x;
        worst = fmax(worst, fabs(y - got) / (g * hl1));
    }
    return worst;
}

int main() {
    srand(11);
    std::vector<int> sizes;
    for (int n = 2; n <= 64; n++) sizes.push_back(n);
    for (int n = 66; n <= 1024; n += 2) sizes.push_back(n);
    for (int n : {96, 97, 320, 384, 512, 640, 1000, 1024, 1536, 2048, 2 * 1009, 4096, 8192}) sizes.push_back(n);
    double worst = 0;
    int worst_n = 0;
    for (int n : sizes) {
        const double r = check(n);
        if (r > worst) { worst = r; worst_n = n; }
    }
    GenFftPlan pl;
    std::vector<float2> tw;
    printf("sizes %zu  worst err / bound %.4f (N = %d)  8193 planned: %s\n", sizes.size(), worst, worst_n,
           gen_fft_plan(8193, pl, tw) ? "yes" : "no");
    const bool ok = worst <= 1.0 && !gen_fft_plan(8193, pl, tw) && !gen_fft_plan(1, pl, tw);
    printf(ok ? "OK\n" : "FAIL\n");
    return ok ? 0 : 1;
}
