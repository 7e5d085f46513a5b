"""A literal restatement of the overhead computer over strings (internal/extender/overhead.go, PodHasReservation in
internal/extender/resourcereservations.go:115-132, GetExecutorSoftReservation in internal/cache/softreservations.go:136-152),
kept independent of the product package: the checker of gp_node_overhead, overhead.encode() and overhead.evaluate().

Pods, lister, ResourceReservations and soft store are described as in k8s_spark_scheduler_b200/overhead.py."""


def pod_to_resources(pod):
    """podToResources (overhead.go:195-209)"""
    cpu = mem = gpu = 0
    for c in pod.get("containers", ()):
        cpu += c.get("cpu", 0)
        mem += c.get("memory", 0)
        gpu += c.get("nvidia.com/gpu", 0)
    for c in pod.get("initContainers", ()):                      # Resources.SetMaxResource
        if c.get("cpu", 0) > cpu:
            cpu = c.get("cpu", 0)
        if c.get("memory", 0) > mem:
            mem = c.get("memory", 0)
        if c.get("nvidia.com/gpu", 0) > gpu:
            gpu = c.get("nvidia.com/gpu", 0)
    return [cpu, mem, gpu]


class OverheadComputer:
    """resourceRequests: map[nodeName]map[UID]PodRequestInfo, driven by FilteringResourceEventHandler{podHasNodeName}"""

    def __init__(self):
        self.resource_requests = {}

    @staticmethod
    def _has_node_name(pod):
        return pod.get("nodeName", "") != ""

    # client-go FilteringResourceEventHandler
    def on_add(self, pod):
        if self._has_node_name(pod):
            self.add_pod_requests(pod)

    def on_update(self, old, new):
        newer, older = self._has_node_name(new), self._has_node_name(old)
        if newer and not older:
            self.add_pod_requests(new)
        elif not newer and older:
            self.delete_pod_requests(old)

    def on_delete(self, pod):
        if self._has_node_name(pod):
            self.delete_pod_requests(pod)

    def _get_or_create(self, node):
        if node not in self.resource_requests:
            self.resource_requests[node] = {}
        return self.resource_requests[node]

    def add_pod_requests(self, pod):                             # :163-174
        self._get_or_create(pod["nodeName"])[pod["uid"]] = (pod["name"], pod["namespace"], pod_to_resources(pod))

    def delete_pod_requests(self, pod):                          # :176-193
        reqs = self._get_or_create(pod["nodeName"])
        if pod["uid"] not in reqs:
            return
        del reqs[pod["uid"]]
        if not reqs:
            del self.resource_requests[pod["nodeName"]]

    def compute_node_overhead(self, node, lister, rrs, soft):    # :120-153 -> (overhead, nonsched, warnings)
        reqs = self.resource_requests.get(node)
        if reqs is None:
            return [0, 0, 0], [0, 0, 0], 0
        overhead, nonsched, warned = [0, 0, 0], [0, 0, 0], 0
        for name, namespace, requests in reqs.values():
            pod = lister.get((namespace, name))
            if pod is None:
                continue
            if not pod_has_reservation(pod, rrs, soft):
                overhead = [a + b for a, b in zip(overhead, requests)]
                if pod.get("schedulerName") == "spark-scheduler":
                    if (pod["namespace"], pod.get("labels", {}).get("spark-app-id", "")) in rrs:
                        warned += 1
                else:
                    nonsched = [a + b for a, b in zip(nonsched, requests)]
        return overhead, nonsched, warned

    def get_overhead_by_node(self, nodes, lister, rrs, soft):   # :105-117
        # Status.Pods values and Reservations keys as sets: the same answers as the reference's scan and map lookup, without
        # its O(k^2) per application of k reserved pods
        rrs = {k: set(v) for k, v in rrs.items()}
        soft = {k: set(v) for k, v in soft.items()}
        overhead, nonsched, warned = {}, {}, 0
        for n in nodes:
            overhead[n], nonsched[n], w = self.compute_node_overhead(n, lister, rrs, soft)
            warned += w
        return overhead, nonsched, warned


def pod_has_reservation(pod, rrs, soft):
    labels = pod.get("labels", {})
    if "spark-app-id" not in labels:
        return False
    app = labels["spark-app-id"]
    rr = rrs.get((pod["namespace"], app))
    if rr is not None and pod["name"] in rr:
        return True
    if labels.get("spark-role", "") == "executor":
        sr = soft.get(app)
        if sr is not None and pod["name"] in sr:
            return True
    return False


def columns(nodes, by_node):
    """{node: [cpu, mem, gpu]} -> three lists in `nodes` order"""
    return tuple([by_node[n][d] for n in nodes] for d in range(3))
