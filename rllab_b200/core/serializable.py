"""Serializable: the pickling contract of rllab's algorithm classes (rllab/core/serializable.py).

A subclass calls `quick_init(self, locals())` first thing in its constructor.  The arguments the constructor was called
with are bound against its signature and kept; pickling stores only them, and unpickling calls the constructor again with
the same arguments.  Device state is therefore never pickled: it is rebuilt by the constructor.
"""
import inspect


class Serializable(object):
    def quick_init(self, locals_):
        """Record the constructor's arguments from its local namespace (called before any other assignment)."""
        if "_ctor_call" in self.__dict__:
            return
        sig = inspect.signature(type(self).__init__)
        args, kwargs = [], {}
        for name, p in list(sig.parameters.items())[1:]:          # skip self
            if p.kind == inspect.Parameter.VAR_POSITIONAL:
                args.extend(locals_[name])
            elif p.kind == inspect.Parameter.VAR_KEYWORD:
                kwargs.update(locals_[name])
            elif p.kind == inspect.Parameter.KEYWORD_ONLY:
                kwargs[name] = locals_[name]
            else:
                args.append(locals_[name])
        sig.bind(self, *args, **kwargs)                          # the recorded call must be a valid call
        self._ctor_call = (tuple(args), kwargs)

    def __getstate__(self):
        args, kwargs = self._ctor_call
        return dict(ctor_args=args, ctor_kwargs=kwargs)

    def __setstate__(self, d):
        fresh = type(self)(*d["ctor_args"], **d["ctor_kwargs"])
        self.__dict__.update(fresh.__dict__)
