"""Mean functions (src/means/*.jl) -- O(N d) host work, exactly as the shim keeps them on the host:
mu = mean(gp.mean, gp.x) (src/GPE.jl:206), dmll_mean! (src/GPE.jl:282-288).  x is (N, d) here."""
import numpy as np


class Mean:
    def get_params(self):
        return []

    def set_params(self, hyp):
        pass

    def num_params(self):
        return len(self.get_params())

    def mean(self, X):
        raise NotImplementedError

    def grad_stack(self, X):
        raise NotImplementedError

    def grad_x(self, X):
        """d mean(x_i) / d x_i as an (N, d) array (the mean's part of the predictive-mean gradient)."""
        raise NotImplementedError


class MeanZero(Mean):                     # mZero.jl
    def mean(self, X):
        return np.zeros(X.shape[0])

    def grad_stack(self, X):
        return np.zeros((X.shape[0], 0))

    def grad_x(self, X):
        return np.zeros(X.shape)

    def spec(self):
        return ("MeanZero",)


class MeanConst(Mean):                    # mConst.jl
    def __init__(self, beta):
        self.beta = float(beta)

    def get_params(self):
        return [self.beta]

    def set_params(self, hyp):
        if len(hyp) != 1:
            raise ValueError("Constant mean function only has 1 parameter")
        self.beta = float(hyp[0])

    def mean(self, X):
        return np.full(X.shape[0], self.beta)

    def grad_stack(self, X):
        return np.ones((X.shape[0], 1))

    def grad_x(self, X):
        return np.zeros(X.shape)

    def spec(self):
        return ("MeanConst", self.beta)


class MeanLin(Mean):                      # mLin.jl
    def __init__(self, beta):
        self.beta = np.asarray(beta, dtype=np.float64).copy()

    def get_params(self):
        return list(self.beta)

    def set_params(self, hyp):
        if len(hyp) != len(self.beta):
            raise ValueError("Linear mean function only has %d parameters" % len(self.beta))
        self.beta = np.asarray(hyp, dtype=np.float64).copy()

    def mean(self, X):
        return X @ self.beta

    def grad_x(self, X):
        return np.broadcast_to(self.beta, X.shape).copy()

    def grad_stack(self, X):
        return np.array(X, dtype=np.float64)

    def spec(self):
        return ("MeanLin", list(self.beta))
