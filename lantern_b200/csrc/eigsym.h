// lantern_b200 -- eigen-decomposition of a small dense symmetric matrix on the host, in double.
//
// Householder reduction to tridiagonal form, then the implicit QL iteration with shifts (the EISPACK tred2 / tql2 pair, as
// published in the public-domain JAMA library).  Used once per index to choose the projected screen's basis (pscreen.cu),
// so it favours plain, deterministic code over speed: the same matrix always gives the same bits.
#pragma once
#include <math.h>
#include <stddef.h>

#include <algorithm>
#include <numeric>
#include <vector>

namespace lb200 {

// a: n x n symmetric, row-major (only read).  On return `val` holds the eigenvalues in descending order and row i of `vec`
// (n x n, row-major) the unit eigenvector of val[i].
inline void eig_symmetric(const std::vector<double>& a, size_t n, std::vector<double>& val, std::vector<double>& vec) {
    std::vector<double> V(a), d(n), e(n);
    auto v = [&](size_t r, size_t c) -> double& { return V[r * n + c]; };
    // ---- tred2: V <- orthogonal Q with Q^T A Q tridiagonal (diagonal d, sub-diagonal e)
    for (size_t j = 0; j < n; ++j)
        d[j] = v(n - 1, j);
    for (size_t i = n - 1; i > 0; --i) {
        double scale = 0.0, h = 0.0;
        for (size_t k = 0; k < i; ++k)
            scale += fabs(d[k]);
        if (scale == 0.0) {
            e[i] = d[i - 1];
            for (size_t j = 0; j < i; ++j) {
                d[j] = v(i - 1, j);
                v(i, j) = 0.0;
                v(j, i) = 0.0;
            }
        } else {
            for (size_t k = 0; k < i; ++k) {
                d[k] /= scale;
                h += d[k] * d[k];
            }
            double f = d[i - 1], g = sqrt(h);
            if (f > 0)
                g = -g;
            e[i] = scale * g;
            h -= f * g;
            d[i - 1] = f - g;
            for (size_t j = 0; j < i; ++j)
                e[j] = 0.0;
            for (size_t j = 0; j < i; ++j) {
                f = d[j];
                v(j, i) = f;
                g = e[j] + v(j, j) * f;
                for (size_t k = j + 1; k <= i - 1; ++k) {
                    g += v(k, j) * d[k];
                    e[k] += v(k, j) * f;
                }
                e[j] = g;
            }
            f = 0.0;
            for (size_t j = 0; j < i; ++j) {
                e[j] /= h;
                f += e[j] * d[j];
            }
            const double hh = f / (h + h);
            for (size_t j = 0; j < i; ++j)
                e[j] -= hh * d[j];
            for (size_t j = 0; j < i; ++j) {
                f = d[j];
                g = e[j];
                for (size_t k = j; k <= i - 1; ++k)
                    v(k, j) -= (f * e[k] + g * d[k]);
                d[j] = v(i - 1, j);
                v(i, j) = 0.0;
            }
        }
        d[i] = h;
    }
    for (size_t i = 0; i + 1 < n; ++i) { // accumulate the transformations
        v(n - 1, i) = v(i, i);
        v(i, i) = 1.0;
        const double h = d[i + 1];
        if (h != 0.0) {
            for (size_t k = 0; k <= i; ++k)
                d[k] = v(k, i + 1) / h;
            for (size_t j = 0; j <= i; ++j) {
                double g = 0.0;
                for (size_t k = 0; k <= i; ++k)
                    g += v(k, i + 1) * v(k, j);
                for (size_t k = 0; k <= i; ++k)
                    v(k, j) -= g * d[k];
            }
        }
        for (size_t k = 0; k <= i; ++k)
            v(k, i + 1) = 0.0;
    }
    for (size_t j = 0; j < n; ++j) {
        d[j] = v(n - 1, j);
        v(n - 1, j) = 0.0;
    }
    v(n - 1, n - 1) = 1.0;
    e[0] = 0.0;
    // ---- tql2 on the transpose W = V^T (the rotations then touch two contiguous rows): W's rows become the eigenvectors
    std::vector<double> W(n * n);
    for (size_t r = 0; r < n; ++r)
        for (size_t c = 0; c < n; ++c)
            W[c * n + r] = V[r * n + c];
    for (size_t i = 1; i < n; ++i)
        e[i - 1] = e[i];
    e[n - 1] = 0.0;
    double f = 0.0, tst1 = 0.0;
    const double eps = 0x1p-52;
    for (size_t l = 0; l < n; ++l) {
        tst1 = std::max(tst1, fabs(d[l]) + fabs(e[l]));
        size_t m = l;
        while (m < n - 1 && !(fabs(e[m]) <= eps * tst1))
            ++m;
        if (m > l) {
            for (int iter = 0; iter < 64; ++iter) {
                double g = d[l];
                double p = (d[l + 1] - g) / (2.0 * e[l]);
                double r = hypot(p, 1.0);
                if (p < 0)
                    r = -r;
                d[l] = e[l] / (p + r);
                d[l + 1] = e[l] * (p + r);
                const double dl1 = d[l + 1];
                double h = g - d[l];
                for (size_t i = l + 2; i < n; ++i)
                    d[i] -= h;
                f += h;
                p = d[m];
                double c = 1.0, c2 = c, c3 = c, s = 0.0, s2 = 0.0;
                const double el1 = e[l + 1];
                for (size_t ii = m; ii-- > l;) {
                    c3 = c2;
                    c2 = c;
                    s2 = s;
                    g = c * e[ii];
                    h = c * p;
                    r = hypot(p, e[ii]);
                    e[ii + 1] = s * r;
                    s = e[ii] / r;
                    c = p / r;
                    p = c * d[ii] - s * g;
                    d[ii + 1] = h + s * (c * g + s * d[ii]);
                    double* w0 = &W[ii * n];
                    double* w1 = &W[(ii + 1) * n];
                    for (size_t k = 0; k < n; ++k) {
                        const double t = w1[k];
                        w1[k] = s * w0[k] + c * t;
                        w0[k] = c * w0[k] - s * t;
                    }
                }
                p = -s * s2 * c3 * el1 * e[l] / dl1;
                e[l] = s * p;
                d[l] = c * p;
                if (!(fabs(e[l]) > eps * tst1))
                    break;
            }
        }
        d[l] += f;
        e[l] = 0.0;
    }
    std::vector<size_t> order(n);
    std::iota(order.begin(), order.end(), 0);
    std::stable_sort(order.begin(), order.end(), [&](size_t x, size_t y) { return d[x] > d[y]; });
    val.resize(n);
    vec.resize(n * n);
    for (size_t i = 0; i < n; ++i) {
        val[i] = d[order[i]];
        std::copy(&W[order[i] * n], &W[order[i] * n] + n, &vec[i * n]);
    }
}

} // namespace lb200
