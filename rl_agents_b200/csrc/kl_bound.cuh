// KL confidence bounds of a Bernoulli mean (rl_agents/utils.py:89-203), shared by olop.cu and mdp_gape.cu.
#pragma once
#include <math.h>

namespace b2 {

// bernoulli_kullback_leibler (utils.py:89-106)
__device__ __forceinline__ double bernoulli_kl(double p, double q) {
    double kl1 = 0.0, kl2 = INFINITY;
    if (p > 0.0 && q > 0.0) kl1 = p * log(p / q);
    if (q < 1.0) kl2 = p < 1.0 ? (1.0 - p) * log((1.0 - p) / (1.0 - q)) : 0.0;
    return kl1 + kl2;
}

// kl_upper_bound(_sum, count, threshold, lower) with eps = 1e-2 (utils.py:123-147) through newton_iteration
// (:150-203) on [mu, 1] (upper) or [0, mu] (lower): start at the midpoint, pull back with weight 0.9 when a step
// leaves the interval, stop on |dx| <= eps or 100 iterations.
__device__ __forceinline__ double kl_bound(double sum, int count, double threshold, bool lower) {
    if (count == 0) return lower ? 0.0 : 1.0;
    const double eps = 1e-2, weight = 0.9;
    const double mu = sum / (double)count;
    const double max_div = threshold / (double)count;
    const double a = lower ? 0.0 : mu, b = lower ? mu : 1.0;
    if (a == b) return a;
    double x = INFINITY, x_next = (a + b) / 2.0;
    int iterations = 0;
    while (fabs(x - x_next) > eps && iterations < 100) {
        ++iterations;
        x = x_next;
        const double f_x = bernoulli_kl(mu, x) - max_div;
        double df_x;
        if (x == 0.0 || x == 1.0)      // Python float division raises ZeroDivisionError (:183-186)
            df_x = (f_x - (bernoulli_kl(mu, x - eps) - max_div)) / eps;
        else
            df_x = (1.0 - mu) / (1.0 - x) - mu / x;
        if (df_x != 0.0) x_next = x - f_x / df_x;
        if (x_next < a) x_next = weight * a + (1.0 - weight) * x;
        else if (x_next > b) x_next = weight * b + (1.0 - weight) * x;
    }
    if (x_next < a) x_next = a;
    if (x_next > b) x_next = b;
    return x_next;
}

__device__ __forceinline__ double kl_upper_bound(double sum, int count, double threshold) {
    return kl_bound(sum, count, threshold, false);
}

}  // namespace b2
