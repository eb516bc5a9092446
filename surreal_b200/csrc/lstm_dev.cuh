// The LSTM cell of RNN-mode PPO (torch.nn.LSTM, gate order i, f, g, o), shared by the learner's sequence kernel
// (lstm.cu) and the persistent recurrent rollout (rollout_rnn.cu), whose results must agree bit for bit with the per-step
// launch chain: one definition of the gate pre-activation sum and of the cell update, so every caller gets the same
// rounding and the same FMA contraction.
#pragma once
#include "common.cuh"

namespace {

__device__ __forceinline__ float sigmoidf_(float x) { return 1.0f / (1.0f + expf(-x)); }

// F.linear(x, w_ih, b_ih) + F.linear(h, w_hh, b_hh): pre_x = x . W_ih^T + b_ih, acc = h . W_hh^T
__device__ __forceinline__ float lstm_gate_pre(float pre_x, float acc, float b_hh) { return pre_x + (acc + b_hh); }

struct LstmGates {
    float i, f, g, o;     // activated gates
};

// Activated gates from the four pre-activations, and the cell update c <- f c + i g, h = o tanh(c).  Returns h.
__device__ __forceinline__ float lstm_cell(float pi, float pf, float pg, float po, float& c, LstmGates& q) {
    q.i = sigmoidf_(pi);
    q.f = sigmoidf_(pf);
    q.g = tanhf(pg);
    q.o = sigmoidf_(po);
    c = q.f * c + q.i * q.g;
    return q.o * tanhf(c);
}

}  // namespace
